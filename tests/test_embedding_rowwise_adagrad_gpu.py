"""Row-wise AdaGrad for embedding-collection tables (Optimizer_t.RowWiseAdaGrad).

Definition, for a table row r that receives gradients in a step, with ev columns:
  g[c]  = (sum of the row's gradient contributions, 1/nnz for mean) * grad_scale / scaler
  s[r] += (1/ev) * sum_c g[c]^2          one fp32 accumulator per row, starting at initial_accu_value
  w[c] -= lr * g[c] / (sqrt(s[r]) + eps)
Rows without gradient are untouched.

The oracle below is written from that definition in fp64 on the per-row gradient sums of
test_embedding_kernels_gpu.py (oracle_reduce), not from the package's CPU path.

Error bound (stated once, used everywhere).  The kernels sum a row's n gradient rows in fp32 in any
order, so every summed column lies within e = (n + 4) u sum|g| of the exact one (u = 2^-24).  Then
  s:  |ds| <= mean_c(2 |g| e + e^2) + (ev + 8) u (|s_old| + mean_c g^2)       (the row's fp32 sum)
  w:  with D = sqrt(s) + eps and dD <= |ds| / (2 sqrt(s)) + 4 u D,
      |d dw| <= lr e / D + lr |g| dD / D^2 + 16 u (|dw| + |w_old| + |w_new|)
bf16 weights may additionally differ by one bf16 ulp of the new weight (stochastic rounding).
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_embedding_kernels_gpu as K  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.enums import Optimizer_t as O  # noqa: E402

U = K.U
RW = O.RowWiseAdaGrad
BF = torch.bfloat16
HP = dict(K.HP, epsilon=2.0 ** -10, initial_accu_value=0.0)
LR = K.LR


# ------------------------------------------------------------------------------------------ oracle
def rowwise_oracle(red, w_old, s_old, hp=HP, lr=LR):
    """(expected w_new - w_old [n, ev], expected s_new [n], bounds of both) of the rows ``red`` touches,
    in fp64; w_old [n, ev], s_old [n] are the rows' values before the step"""
    uniq, G, A, n = red
    scaler, eps = hp.get("scaler", 1.0), hp["epsilon"]
    g = G / scaler
    e = (n.view(-1, 1) + 4).double() * U * A / scaler
    s = s_old.double() + (g * g).mean(1)
    D = s.sqrt() + eps
    dw = -lr * g / D.view(-1, 1)
    ds = (2 * g.abs() * e + e * e).mean(1) + (g.shape[1] + 8) * U * (s_old.double().abs() + (g * g).mean(1))
    dD = ds / (2 * s.sqrt().clamp(min=1e-300)) + 4 * U * D
    tw = lr * e / D.view(-1, 1) + lr * g.abs() * (dD / (D * D)).view(-1, 1) \
        + 16 * U * (dw.abs() + w_old.double().abs() + (w_old.double() + dw).abs())
    return dw, s, tw, ds


def check_rowwise(what, case, tab, s, new, hp=HP, lr=LR, grad_scale=1.0, bf16=False):
    """kernel / CPU result ``new`` = (w, s) against the oracle; rows no pair touches must not change"""
    P = case.pitch
    red = K.oracle_reduce(case, grad_scale)
    uniq = red[0]
    w_old = tab.view(-1, P)[uniq].double()
    dw, s_ref, tw, ts = rowwise_oracle(red, w_old, s[uniq], hp, lr)
    w_new, s_new = new[0].cpu().view(-1, P), new[1].cpu()
    if bf16:
        tw = tw + K.bf16_ulp(w_old + dw)
    K.assert_close_bound(f"{what} dw", w_new[uniq].double() - w_old, dw, tw)
    K.assert_close_bound(f"{what} s", s_new[uniq], s_ref, ts)
    keep = torch.ones(tab.numel() // P, dtype=torch.bool)
    keep[uniq] = False
    assert torch.equal(w_new[keep], tab.view(-1, P)[keep]), f"{what}: untouched w rows changed"
    assert torch.equal(s_new[keep], s[keep]), f"{what}: untouched s rows changed"


def init_rowwise(rows, pitch, gen, wdt=torch.float32):
    tab = (torch.randn(rows * pitch, generator=gen) * 0.1).to(wdt)
    s = torch.rand(rows, generator=gen) * 0.5 + 0.01
    return tab, s


# ------------------------------------------------------------------------------------------ CPU: oracle
def test_oracle_matches_package_cpu_path():
    """sparse_opt_reference / update_rows (the CPU path of backward_accum + update) agree with the
    oracle on a case with every lookup feature, loss scaler and grad_scale != 1"""
    gen = torch.Generator().manual_seed(1)
    case = K.features_case(8, torch.float32, gen, batch=40)
    tab, s = init_rowwise(case.rows, case.pitch, gen)
    hp = dict(HP, scaler=4.0)
    t, a = tab.clone(), s.clone()
    ws = E.UniqueWorkspace(case.pairs, case.pitch, torch.device("cpu"))
    E.backward_accum(case.lookups, None, t, case.pitch, case.keys, case.grads, case.batch, ws, 0.5,
                     nnz_bufs=case.nnz)
    E.update(RW, t, a, None, case.pitch, ws, hp, torch.tensor([LR]), torch.tensor([3], dtype=torch.int32))
    check_rowwise("cpu", case, tab, s, (t, a), hp=hp, grad_scale=0.5)


def _expected(case, tab, s, variant):
    """fp32 results of three wrong rules: 'sum' (s += sum_c g^2), 'elementwise' (a state per
    element) and 'early' (s updated from the row's first contribution only)"""
    P = case.pitch
    uniq, G, _, n = K.oracle_reduce(case)
    w, st = tab.clone().view(-1, P), s.clone()
    eps = HP["epsilon"]
    s0 = s[uniq].double()
    if variant == "sum":
        sn = s0 + (G * G).sum(1)
        w[uniq] = (w[uniq].double() - LR * G / (sn.sqrt() + eps).view(-1, 1)).float()
    elif variant == "elementwise":
        sn = s0.view(-1, 1) + G * G
        w[uniq] = (w[uniq].double() - LR * G / (sn.sqrt() + eps)).float()
        sn = sn.mean(1)
    else:
        keys = case.keys[0].view(case.batch, -1)
        first = torch.stack([case.grads[0].view(case.batch, P)[(keys == r).any(1).nonzero()[0, 0]].double()
                             for r in uniq])
        sn = s0 + (first * first).mean(1)
        w[uniq] = (w[uniq].double() - LR * G / (sn.sqrt() + eps).view(-1, 1)).float()
    st[uniq] = sn.float()
    return w.view(-1), st


def test_oracle_rejects_wrong_rules():
    gen = torch.Generator().manual_seed(2)
    case = K.single_case(K.class_keys(512, 8, 3000, gen), 512, 8, 16, 3000, torch.float32, gen)
    tab, s = init_rowwise(3000, 16, gen)
    uniq, G, _, n = K.oracle_reduce(case)
    dw, s_ref, _, _ = rowwise_oracle((uniq, G, _, n), tab.view(-1, 16)[uniq], s[uniq])
    good_w, good_s = tab.clone().view(-1, 16), s.clone()
    good_w[uniq] = (tab.view(-1, 16)[uniq].double() + dw).float()
    good_s[uniq] = s_ref.float()
    check_rowwise("exact", case, tab, s, (good_w.view(-1), good_s))
    for variant in ("sum", "elementwise", "early"):
        with pytest.raises(AssertionError, match="outside the bound"):
            check_rowwise(variant, case, tab, s, _expected(case, tab, s, variant))


# ------------------------------------------------------------------------------------------ CPU: API
def test_rowwise_is_rejected_outside_embedding_collections():
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.sok import OptimizerWrapper
    rw = hugectr.CreateOptimizer(RW, initial_accu_value=0.1, epsilon=1e-8)
    solver = hugectr.CreateSolver(batchsize=8, batchsize_eval=8, vvgpu=[[0]], use_embedding_collection=True)
    reader = hugectr.DataReaderParams(data_reader_type=hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.1"],
                                      eval_source="synthetic:1.1", check_type=hugectr.Check_t.Non, slot_size_array=[10])
    with pytest.raises(ValueError, match=r"EmbeddingTableConfig\(opt_params=...\)"):
        hugectr.Model(solver, reader, rw, comm=Comm.single(torch.device("cpu")))
    with pytest.raises(ValueError, match=r"EmbeddingTableConfig\(opt_params=...\)"):
        hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 1, 8, "sum", "e", "d",
                                [10], optimizer=rw)
    with pytest.raises(ValueError, match=r"EmbeddingTableConfig\(opt_params=...\)"):
        OptimizerWrapper(RW)


def test_graph_json_of_the_optimizer_round_trips():
    from hugectr_b200.solver import CreateOptimizer, OptParamsPy
    o = CreateOptimizer(RW, initial_accu_value=0.25, epsilon=1e-6)
    j = o.to_json()
    assert j["type"] == "RowWiseAdaGrad" and j["adagrad_hparam"] == {"initial_accu_value": 0.25, "epsilon": 1e-6}
    b = OptParamsPy.from_json(j)
    assert (b.optimizer_type, b.initial_accu_value, b.epsilon) == (RW, 0.25, 1e-6)


def _mixed_collection(dev, opt_c=None):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    ts = [EmbeddingTableConfig("rw", 100, 16, opt_params=CreateOptimizer(RW, initial_accu_value=0.1, epsilon=1e-6)),
          EmbeddingTableConfig("ada", 80, 16, opt_params=CreateOptimizer(O.AdaGrad, initial_accu_value=0.2)),
          EmbeddingTableConfig("sgd", 60, 16, opt_params=CreateOptimizer(O.SGD)),
          EmbeddingTableConfig("rwdp", 40, 16, opt_params=CreateOptimizer(RW, initial_accu_value=0.1, epsilon=1e-6))]
    cfg.embedding_lookup(ts, ["d0", "d1", "d2", "d3"], "emb", ["sum", "mean", "sum", "sum"])
    cfg.shard([[1, 1, 1, 1]], [("mp", ["rw", "ada"]), ("dp", ["sgd", "rwdp"])])
    return EmbeddingCollection(cfg, 16, {"d0": 3, "d1": 2, "d2": 1, "d3": 2}, dev, torch.float32, Comm.single(dev),
                               CreateOptimizer(O.Adam), seed=1)


def test_mixed_optimizers_of_one_width_keep_their_own_optimizer():
    e = _mixed_collection(torch.device("cpu"))
    by_table = {sl["table"]: g for g in e.groups for sl in g.table_slices}
    assert by_table["rw"].opt.optimizer_type == RW and [s["table"] for s in by_table["rw"].table_slices] == ["rw"]
    assert by_table["ada"].opt.optimizer_type == O.AdaGrad
    assert by_table["sgd"].opt.optimizer_type == O.SGD
    assert by_table["rwdp"].opt.optimizer_type == RW and by_table["rwdp"].kind == "dp"
    for name in ("rw", "rwdp"):
        g = by_table[name]
        assert g.s0.dtype == torch.float32 and g.s0.numel() == g.rows and g.s1 is None
        assert bool((g.s0 == 0.1).all())


def test_state_is_fp32_per_row_even_with_bf16_state():
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig("t", 50, 8, weight_dtype="bf16", opt_params=CreateOptimizer(RW))],
                         ["d"], "emb", ["sum"])
    cpu = torch.device("cpu")
    e = EmbeddingCollection(cfg, 4, {"d": 1}, cpu, torch.float32, Comm.single(cpu), CreateOptimizer(O.SGD),
                            state_dtype=BF)
    assert e.groups[0].s0.dtype == torch.float32
    assert e.memory_bytes() == 50 * 8 * 2 + 50 * 4


# ------------------------------------------------------------------------------------------ CPU: model
def _tiny_model(wdt, seed=7, dyn=False, table_opt="rowwise"):
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    sizes, hot = [50, 40, 30, 20], [2, 1, 1, 2]
    solver = hugectr.CreateSolver(model_name="rowwise", seed=seed, batchsize=32, batchsize_eval=32,
                                  vvgpu=[[0]], lr=0.05, use_mixed_precision=False, use_cuda_graph=False,
                                  use_embedding_collection=True, warmup_steps=1, max_eval_batches=1)
    reader = hugectr.DataReaderParams(
        data_reader_type=hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.1"], eval_source="synthetic:1.1",
        check_type=hugectr.Check_t.Non, slot_size_array=sizes,
        async_param=hugectr.AsyncParam(1, 16, shuffle=False, multi_hot_reader=True, is_dense_float=True))
    opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, hugectr.Update_t.Global, initial_accu_value=0.0,
                                  epsilon=1e-8)
    m = hugectr.Model(solver, reader, opt, comm=Comm.single(torch.device("cpu")))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=13, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam(f"data{i}", hot[i], True, 1)
                                                        for i in range(4)]))
    to = hugectr.CreateOptimizer(RW, initial_accu_value=0.01, epsilon=1e-8) if table_opt == "rowwise" else None
    tables = [hugectr.EmbeddingTableConfig(name=str(i), max_vocabulary_size=-1 if (dyn and i == 1) else sizes[i],
                                           ev_size=8, weight_dtype=wdt, opt_params=to, init_capacity=16)
              for i in range(4)]
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(table_config=tables, bottom_name=[f"data{i}" for i in range(4)],
                         top_name="sparse_embedding", combiner=["sum", "sum", "mean", "sum"])
    ebc.shard([[1, 1, 1, 1]], [("mp", ["0", "1", "2"]), ("dp", ["3"])])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["dense"], ["mlp1"], num_outputs=[16, 8],
                             act_type=hugectr.Activation_t.Relu))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["sparse_embedding", "mlp1"], ["concat1"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.MLP, ["concat1"], ["mlp2"], num_outputs=[16, 1],
                             activations=[hugectr.Activation_t.Relu, hugectr.Activation_t.Non]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["mlp2", "label"], ["loss"]))
    m.compile()
    return m


@pytest.mark.parametrize("wdt,dyn", [("fp32", False), ("bf16", False), ("fp32", True), ("bf16", True)])
def test_rowwise_model_trains_round_trips_and_resumes(tmp_path, wdt, dyn):
    import json
    a = _tiny_model(wdt, dyn=dyn)
    e = a.ebcs_train[0]
    assert all(g.rowwise for g in e.groups) and sorted(g.kind for g in e.groups) == ["dp", "mp"]
    pool = a.reader_train.pool
    t0 = [g.table.clone() for g in e.groups]
    s0 = [g.s0.clone() for g in e.groups]
    pre = str(tmp_path / "snap")
    losses = []
    for i in range(7):
        a.train_on_host_batch(pool[i % len(pool)])
        losses.append(a.get_current_loss())
        if i == 4:
            a.save_params_to_files(pre, 5)
    assert all(math.isfinite(x) for x in losses)
    for g, t, s in zip(e.groups, t0, s0):
        assert not torch.equal(t, g.table), g.kind
        if not dyn:
            assert bool((g.s0 >= s).all()) and bool((g.s0 > s).any()), g.kind
    if dyn:   # more distinct keys than the 16 initial rows: the model grew the dynamic table
        assert any(sl["rows"] > 16 for g in e.groups for sl in g.table_slices if sl["dynamic"])
    # 4 B of state per row
    assert e.memory_bytes() == sum(g.table.numel() * g.table.element_size() + 4 * g.rows for g in e.groups)
    # graph JSON
    a.graph_to_json(str(tmp_path / "g.json"))
    tj = [l for l in json.load(open(tmp_path / "g.json"))["layers"] if l["type"] == "EmbeddingCollection"][0]
    assert all(t["optimizer"]["type"] == "RowWiseAdaGrad" for t in tj["tables"])
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]],
                                  use_embedding_collection=True, use_cuda_graph=False)
    m2 = hugectr.Model(solver, a.reader_params, a.opt_params, comm=Comm.single(torch.device("cpu")))
    m2.construct_from_json(str(tmp_path / "g.json"))
    assert all(t.opt_params.optimizer_type == RW and t.opt_params.initial_accu_value == 0.01
               for t in m2.ebc_configs[0].tables())
    # dump -> load -> dump is byte-identical, state included
    d1 = {str(i): e.dump_table_local(str(i)) for i in range(4)}
    b = _tiny_model(wdt, seed=99, dyn=dyn)
    for name, parts in d1.items():
        for keys, w, col0, sts, kind in parts:
            assert len(sts) == 2 and sts[1] is None and sts[0].shape == w.shape
            b.ebcs_train[0].load_table_rows(name, keys, w, sts)
    for name, parts in d1.items():
        for x, y in zip(parts, b.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(x[0], y[0])
            assert x[1].numpy().tobytes() == y[1].numpy().tobytes()
            assert x[3][0].numpy().tobytes() == y[3][0].numpy().tobytes()
    if not dyn:
        # resume from the step-5 snapshot: bit-identical continuation.  (A dynamic table does not resume
        # bit-identically with any optimizer: keys first seen after the snapshot start from initial values
        # drawn for the arena rows they land in, and those differ between the grown and the reloaded table.)
        c = _tiny_model(wdt)
        assert c.resume(pre) == 5
        for i in range(5, 7):
            c.train_on_host_batch(pool[i % len(pool)])
        assert float((a.arena.weights - c.arena.weights).abs().max()) == 0.0
        for name in d1:
            for pa, pc in zip(e.dump_table_local(name), c.ebcs_train[0].dump_table_local(name)):
                assert torch.equal(pa[1], pc[1]) and torch.equal(pa[3][0], pc[3][0])


def test_adagrad_checkpoints_convert_both_ways(tmp_path):
    """an AdaGrad checkpoint loads into row-wise tables as the row mean of its state, and a row-wise
    checkpoint loads into AdaGrad tables as every element holding its row's value"""
    ada = _tiny_model("fp32", table_opt="adagrad")
    for i in range(3):
        ada.train_on_host_batch(ada.reader_train.pool[i])
    pre = str(tmp_path / "ada")
    ada.save_params_to_files(pre, 3)
    rw = _tiny_model("fp32", seed=5)
    rw.embedding_load(pre + "_ebc_3")
    for name in ("0", "1", "2", "3"):
        for pa, pr in zip(ada.ebcs_train[0].dump_table_local(name), rw.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pa[1], pr[1])
            assert torch.equal(pr[3][0], pa[3][0].double().mean(1, keepdim=True).float().expand_as(pa[3][0]))
    rw.save_params_to_files(pre + "rw", 3)
    back = _tiny_model("fp32", seed=6, table_opt="adagrad")
    back.embedding_load(pre + "rw_ebc_3")
    for name in ("0", "1", "2", "3"):
        for pr, pb in zip(rw.ebcs_train[0].dump_table_local(name), back.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pr[3][0], pb[3][0])


def test_planner_accounts_for_row_state():
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    from hugectr_b200.tools.planner import plan_tables
    gb = plan_tables(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, 128, 1, weight_bytes=2, state_bytes=0,
                     state_row_bytes=4)[2]["memory_gb"][0]
    rows = sum(CRITEO_TB_TABLE_SIZES)
    assert gb == pytest.approx(rows * (128 * 2 + 4) / 1e9)
    assert plan_tables(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, 128, 1)[2]["memory_gb"][0] == \
        pytest.approx(rows * 128 * 8 / 1e9)


# ========================================================================================== GPU
def run_rowwise(case, tab, s, path="fused", hp=HP, lr=LR, grad_scale=1.0, ws=None, dev_state=None, **ws_kw):
    (t, a, _), ws = K.run_step(case, RW, tab, s, None, path=path, hp=hp, lr=lr, grad_scale=grad_scale, ws=ws,
                               dev_state=dev_state, **ws_kw)
    return (t, a), ws


WIDTHS = [4, 8, 12, 64, 124, 128, 132, 256, 516, 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", WIDTHS)
@pytest.mark.parametrize("gdt", [torch.float32, BF])
@pytest.mark.parametrize("wdt", [torch.float32, BF])
def test_fused_row_classes_and_widths(pitch, gdt, wdt):
    """rows occurring 1..5, 64, 65, 512, 513 and 1025 times (light, medium and heavy rows with 1-3
    chunks) at every width class of the fused kernels, fp32 / bf16 gradients and weights"""
    gen = torch.Generator().manual_seed(pitch)
    case = K.single_case(K.class_keys(512, 8, 4000, gen), 512, 8, pitch, 4000, gdt, gen)
    tab, s = init_rowwise(case.rows, pitch, gen, wdt)
    new, ws = run_rowwise(case, tab, s)
    check_rowwise(f"fused ev={pitch}", case, tab, s, new, bf16=wdt == BF)
    K.assert_ws_clean(ws)


ACCUM = [1, 3, 6, 11, 128, 258]


@pytest.mark.gpu
@pytest.mark.parametrize("wdt", [torch.float32, BF])
@pytest.mark.parametrize("pitch", ACCUM)
def test_accumulate_path_with_lookup_features(pitch, wdt):
    """emb_update_kernel (float4 and scalar widths) after backward_accum: mean combiners with variable
    nnz and padding, a row-sharded lookup, two source buffers, grad_scale and scaler != 1"""
    gen = torch.Generator().manual_seed(pitch)
    case = K.features_case(pitch, torch.float32, gen)
    tab, s = init_rowwise(case.rows, pitch, gen, wdt)
    hp = dict(HP, scaler=4.0)
    new, ws = run_rowwise(case, tab, s, path="accum", hp=hp, grad_scale=0.5)
    check_rowwise(f"accum ev={pitch}", case, tab, s, new, hp=hp, grad_scale=0.5, bf16=wdt == BF)
    K.assert_ws_clean(ws)


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", [128, 516])
def test_fused_lookup_features(pitch):
    gen = torch.Generator().manual_seed(pitch + 1)
    case = K.features_case(pitch, BF, gen)
    tab, s = init_rowwise(case.rows, pitch, gen)
    hp = dict(HP, scaler=4.0)
    new, ws = run_rowwise(case, tab, s, hp=hp, grad_scale=0.5, key_dtype=torch.int64)
    check_rowwise(f"fused features ev={pitch}", case, tab, s, new, hp=hp, grad_scale=0.5)
    K.assert_ws_clean(ws)


@pytest.mark.gpu
def test_small_heavy_caps_fall_back_to_the_medium_list():
    """heavy rows beyond 2 scratch rows / 3 chunk items take the warp-per-row kernel; two steps on one
    workspace, clean after each"""
    gen = torch.Generator().manual_seed(4)
    pitch = 516
    tab, s = init_rowwise(3000, pitch, gen)
    ws, state = None, None
    for counts in ([70, 65, 1100, 66, 5, 3, 1], [1025, 600, 65, 70, 64, 2]):
        case = K.single_case(K.class_keys(512, 16, 3000, gen, counts), 512, 16, pitch, 3000, torch.float32, gen)
        state, ws = run_rowwise(case, tab, s, ws=ws, dev_state=(state[0], state[1], None) if state else None,
                                max_heavy_rows=2, max_heavy_items=3)
        check_rowwise("small caps", case, tab, s, state)
        K.assert_ws_clean(ws)
        tab, s = state[0].cpu(), state[1].cpu()


@pytest.mark.gpu
def test_row_with_more_than_4096_chunks():
    gen = torch.Generator().manual_seed(6)
    batch, hot, pitch = 16500, 128, 4
    keys = torch.full((batch * hot,), 7, dtype=torch.int64)
    keys[torch.randperm(keys.numel(), generator=gen)[:3000]] = torch.randint(8, 900, (3000,), generator=gen)
    grads = torch.randint(-2, 3, (batch * pitch,), generator=gen).float() / 16
    case = K.Case([K.lookup(0, 1000, 0, 0, hot, pitch, pitch)], pitch, batch, [keys], [grads])
    tab, s = init_rowwise(1000, pitch, gen)
    new, ws = run_rowwise(case, tab, s)
    check_rowwise("2.1 M-occurrence row", case, tab, s, new)
    K.assert_ws_clean(ws)


@pytest.mark.gpu
@pytest.mark.parametrize("path,pitch", [("fused", 128), ("fused", 1024), ("accum", 128), ("accum", 12)])
def test_bf16_exact_case_bits_match_the_mirror(path, pitch):
    """every column's gradient is +-2^-5: light rows occur once, 20 medium rows 8 times and a heavy
    row 1024 times, always with +2^-5; initial_accu_value = 0 and epsilon = 0.  Then s = k^2 2^-10
    with k in {1, 8, 1024}, f = lr / sqrt(s) and every w - f g are exact in fp32, so the stored bf16
    bits must equal sr_round_bf16 of them"""
    gen = torch.Generator().manual_seed(pitch)
    rows, batch, hot = 4000, 1500, 2
    keys = K.class_keys(batch, hot, rows, gen, [1] * 1200 + [8] * 20 + [1024])
    sign = torch.randint(0, 2, (batch, 1), generator=gen).float() * 2 - 1
    grads = (sign * torch.ones(batch, pitch) * 2.0 ** -5)
    # the medium and heavy rows' occurrences all carry +2^-5
    vals, cnt = keys[keys >= 0].unique(return_counts=True)
    grads[torch.isin(keys.view(batch, hot), vals[cnt > 1]).any(1)] = 2.0 ** -5
    case = K.single_case(keys, batch, hot, pitch, rows, torch.float32, gen)
    case.grads = [grads.reshape(-1)]
    tab = (torch.randint(-2048, 2049, (rows * pitch,), generator=gen).float() / 4096).to(BF)
    s = torch.zeros(rows)
    lr, seed, step = 2.0 ** -4, 0xBEEF, 9
    hp = dict(HP, epsilon=0.0, sr_seed=seed)
    uniq, G, _, n = K.oracle_reduce(case)
    assert int((n == 8).sum()) == 20 and int((n == 1024).sum()) == 1
    f = lr / (G * G).mean(1).sqrt()
    w = tab.double().view(-1, pitch)[uniq] - f.view(-1, 1) * G
    assert torch.equal(w.float().double(), w), "case is not exact in fp32"
    idx = uniq.view(-1, 1) * pitch + torch.arange(pitch).view(1, -1)
    exp = tab.clone().view(-1, pitch)
    exp[uniq] = E.sr_round_bf16(w.float(), seed, step, idx)
    (t, a, _), _ = K.run_step(case, RW, tab, s, None, path=path, hp=hp, lr=lr, step=step)
    got = t.cpu().view(-1, pitch)
    bad = (got.view(torch.int16) != exp.view(torch.int16)).any(1)
    assert not bool(bad.any()), f"{path} ev={pitch}: {int(bad.sum())} rows differ from the mirror"
    assert torch.equal(a.cpu()[uniq].double(), (G * G).mean(1))


@pytest.mark.gpu
@pytest.mark.parametrize("pitch", [6, 128])
def test_dp_update_against_the_oracle(pitch):
    """the row rule on an all-reduced dense gradient: touched rows against the oracle, all-zero rows
    untouched, the gradient zeroed"""
    gen = torch.Generator().manual_seed(pitch)
    rows = 300
    G = torch.randn(rows, pitch, generator=gen).double() * 0.1
    G[torch.randperm(rows, generator=gen)[:100]] = 0
    tab, s = init_rowwise(rows, pitch, gen)
    touched = (G != 0).any(1)
    uniq = touched.nonzero().view(-1)
    wg = G.float().reshape(-1).cuda()
    t, a = tab.cuda(), s.cuda()
    hp = dict(HP, scaler=2.0)
    E.dp_rowwise_update(t, a, wg, pitch, hp, torch.tensor([LR], device="cuda"))
    torch.cuda.synchronize()
    red = (uniq, G.float().double()[uniq], G.abs()[uniq], torch.zeros(uniq.numel(), dtype=torch.long))
    dw, s_ref, tw, ts = rowwise_oracle(red, tab.view(-1, pitch)[uniq].double(), s[uniq], hp)
    K.assert_close_bound("dp dw", t.cpu().view(-1, pitch)[uniq].double() - tab.view(-1, pitch)[uniq].double(), dw, tw)
    K.assert_close_bound("dp s", a.cpu()[uniq], s_ref, ts)
    assert torch.equal(t.cpu().view(-1, pitch)[~touched], tab.view(-1, pitch)[~touched])
    assert torch.equal(a.cpu()[~touched], s[~touched])
    assert int((wg != 0).sum()) == 0


@pytest.mark.gpu
def test_collection_steps_match_the_cpu_path():
    """a collection with row-wise (mp and dp), AdaGrad and SGD tables: three GPU steps equal the CPU
    collection's within tolerance, and a CUDA-graph replay of the backward equals the eager step"""
    g, c = _mixed_collection(torch.device("cuda")), _mixed_collection(torch.device("cpu"))
    for gg, cg in zip(g.groups, c.groups):
        cg.table.copy_(gg.table.cpu())
    gen = torch.Generator().manual_seed(0)
    lr_c, st_c = torch.tensor([0.05]), torch.tensor([1], dtype=torch.int32)
    lr_g, st_g = lr_c.cuda(), st_c.cuda()

    def batch():
        keys = torch.cat([torch.randint(0, v, (16 * h,), generator=gen)
                          for v, h in ((100, 3), (80, 2), (60, 1), (40, 2))]).int()
        grad = torch.randn(c.top_grad["emb"].shape, generator=gen) * 0.1
        return keys, grad

    def step(e, keys, grad, lr, st):
        e.set_keys(keys.to(e.device))
        e.forward()
        e.top_grad["emb"].copy_(grad.to(e.device))
        e.backward(lr, st)

    for _ in range(3):
        keys, grad = batch()
        step(g, keys, grad, lr_g, st_g)
        step(c, keys, grad, lr_c, st_c)
        torch.cuda.synchronize()
        for gg, cg in zip(g.groups, c.groups):
            torch.testing.assert_close(gg.table.cpu(), cg.table, rtol=1e-3, atol=2e-5)
            if gg.s0 is not None:
                torch.testing.assert_close(gg.s0.cpu(), cg.s0, rtol=1e-4, atol=1e-7)
    # CUDA graph of one step against the same step run eagerly from the same state
    keys, grad = batch()
    snap = [(gg.table.clone(), None if gg.s0 is None else gg.s0.clone()) for gg in g.groups]
    step(g, keys, grad, lr_g, st_g)
    torch.cuda.synchronize()
    eager = [(gg.table.clone(), None if gg.s0 is None else gg.s0.clone()) for gg in g.groups]
    for gg, (t, s) in zip(g.groups, snap):
        gg.table.copy_(t)
        if s is not None:
            gg.s0.copy_(s)
    g.set_keys(keys.cuda())
    g.top_grad["emb"].copy_(grad.cuda())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            g.forward()
            g.backward(lr_g, st_g)
    torch.cuda.current_stream().wait_stream(side)
    for gg, (t, s) in zip(g.groups, snap):
        gg.table.copy_(t)
        if s is not None:
            gg.s0.copy_(s)
    g.top_grad["emb"].copy_(grad.cuda())
    graph.replay()
    torch.cuda.synchronize()
    for gg, (t, s) in zip(g.groups, eager):
        assert torch.equal(gg.table, t)
        if s is not None:
            assert torch.equal(gg.s0, s)
    g.check_overflow()


@pytest.mark.gpu
@pytest.mark.parametrize("wdt", ["fp32", "bf16"])
def test_model_cuda_graph_equals_eager(wdt):
    """DLRM-DCNv2 with row-wise AdaGrad tables: six CUDA-graph training steps equal six eager ones"""
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    kw = dict(batchsize=128, num_gpus=1, table_sizes=[5000, 300], multi_hot=[3, 1], ev_size=128,
              bottom=(64, 128), top=(128, 1), projection_dim=64, cross_layers=1, lr=0.01, mixed=True,
              embedding_optimizer="rowwise_adagrad", weight_dtype=wdt)
    a = build_dlrm_dcnv2(use_cuda_graph=True, comm=Comm(torch.device("cuda")), **kw)
    b = build_dlrm_dcnv2(use_cuda_graph=False, comm=Comm(torch.device("cuda")), **kw)
    a.compile(); b.compile()
    b.arena.load_flat(a.arena.dump_flat())
    for ga, gb in zip(a.ebcs_train[0].groups, b.ebcs_train[0].groups):
        assert ga.rowwise and ga.s0.dtype == torch.float32
        gb.table.copy_(ga.table)
        gb.s0.copy_(ga.s0)
    for i in range(6):
        hb = a.reader_train.pool[i % 4]
        a.train_on_host_batch(hb); b.train_on_host_batch(hb)
    torch.cuda.synchronize()
    torch.testing.assert_close(a.arena.weights, b.arena.weights, rtol=1e-3, atol=1e-4)
    for ga, gb in zip(a.ebcs_train[0].groups, b.ebcs_train[0].groups):
        assert bool((ga.s0 > 0).any())
        torch.testing.assert_close(ga.s0, gb.s0, rtol=1e-3, atol=1e-9)
        torch.testing.assert_close(ga.table.float(), gb.table.float(), rtol=2e-2, atol=1e-4)


# ------------------------------------------------------------------------------------------ emulated ranks
def _emu_body(plan, fused, c):
    """one collection per emulated rank (parallel/emu.py) with row-wise AdaGrad on every table, three
    steps against one process holding the whole batch.  Table-wise, row-sharded and data-parallel
    tables must equal the single process (weights and row accumulators); a column-split table keeps
    one accumulator per column slice, so each slice is checked against the oracle applied with the
    slice's own width (one step)"""
    import dist_worker as W
    from hugectr_b200.embedding.collection import EmbeddingCollection
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    world, rank, dev = c.world_size, c.rank, c.device
    cpu = torch.device("cpu")
    b, lr_v, eps, init = 32, 0.05, 1e-6, 0.1
    cfg, sizes, hot, ev = W.make_cfg(world, plan)
    opt = CreateOptimizer(RW, initial_accu_value=init, epsilon=eps)
    e = EmbeddingCollection(cfg, b, hot, dev, torch.float32, c, opt, seed=1, fused=fused)
    assert bool(e.fused) == (fused and world > 1)
    assert all(g.rowwise for g in e.groups)
    ref = EmbeddingCollection(W.make_cfg(1, "none")[0], b * world, hot, cpu, torch.float32, Comm.single(cpu), opt,
                              seed=1)
    gen = torch.Generator().manual_seed(5)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(5)}
    for n, w in full.items():
        k = torch.arange(w.shape[0])
        e.load_table_rows(n, k, w)
        ref.load_table_rows(n, k, w)
    lr, st = torch.tensor([lr_v]), torch.tensor([1], dtype=torch.int32)
    lr_d, st_d = lr.to(dev), st.to(dev)
    split = {n for n in full if e.placement[n].col_factor > 1}
    steps = 1 if split else 3
    for it in range(steps):
        gk = [torch.randint(0, sizes[i], (b * world, h), generator=gen) for i, h in enumerate(hot.values())]
        grad = torch.randn(b * world, 5 * ev, generator=gen) * 0.1
        e.set_keys(torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in gk]).int().to(dev))
        ref.set_keys(torch.cat([k.reshape(-1) for k in gk]).int())
        e.forward(); ref.forward()
        e.top_grad["emb"].copy_(grad[rank * b:(rank + 1) * b].to(dev))
        ref.top_grad["emb"].copy_(grad)
        e.backward(lr_d, st_d); ref.backward(lr, st)
        if dev.type == "cuda":
            torch.cuda.synchronize()
        c.barrier()
    for n in full:
        rk, rw, _, rs, _ = ref.dump_table_local(n)[0]
        for (k, w, c0, sts, kind) in e.dump_table_local(n):
            wd = w.shape[1]
            assert sts[1] is None and sts[0].shape == w.shape
            if n not in split:
                assert (w - rw[k][:, c0:c0 + wd]).abs().max().item() < 2e-4, f"rank {rank} table {n} w"
                torch.testing.assert_close(sts[0], rs[0][k][:, c0:c0 + wd], rtol=1e-4, atol=1e-7)
                continue
            # the slice [c0, c0 + wd) of a sum-combined table, one step: per-row fp64 sums of its columns
            ti = int(n)
            rows = gk[ti].reshape(-1)
            g = grad[:, ti * ev + c0:ti * ev + c0 + wd].double().repeat_interleave(hot[f"d{ti}"], 0)
            uniq, inv = torch.unique(rows, return_inverse=True)
            G = torch.zeros(uniq.numel(), wd, dtype=torch.float64).index_add_(0, inv, g)
            A = torch.zeros_like(G).index_add_(0, inv, g.abs())
            red = (uniq, G, A, torch.bincount(inv))
            w0 = full[n][:, c0:c0 + wd]
            dw, s_ref, tw, ts = rowwise_oracle(red, w0[uniq].double(), torch.full((uniq.numel(),), init),
                                               dict(epsilon=eps), lr_v)
            pos = torch.searchsorted(k, uniq)
            K.assert_close_bound(f"rank {rank} slice {c0} dw", w[pos].double() - w0[uniq].double(), dw, tw)
            K.assert_close_bound(f"rank {rank} slice {c0} s", sts[0][pos, 0], s_ref, ts)
            keep = torch.ones(k.numel(), dtype=torch.bool)
            keep[pos] = False
            assert torch.equal(w[keep], w0[k[keep]]) and bool((sts[0][keep] == init).all())
            # and the slice's own accumulator differs from the unsplit table's
            assert not torch.allclose(sts[0][pos, 0], rs[0][uniq, 0], rtol=1e-3)
    c.barrier()


@pytest.mark.parametrize("plan,world", [("mixed", 2), ("mixed", 3), ("mixed", 4), ("column", 2)])
@pytest.mark.parametrize("fused", [False, True], ids=["collective", "fused"])
def test_emu_ranks_equal_one_process_cpu(plan, world, fused):
    """2-4 emulated ranks on the CPU, on the collective path and with the fused (peer-store) data flow
    forced: a table-wise, a row-sharded and a data-parallel plan equal one process; a column factor of
    2 matches the oracle per column slice"""
    from hugectr_b200.parallel.emu import run_ranks
    run_ranks(world, lambda c: _emu_body(plan, fused, c), device=torch.device("cpu"),
              p2p="force" if fused else True)


@pytest.mark.gpu
@pytest.mark.parametrize("plan,world", [("mixed", 2), ("mixed", 4), ("column", 2), ("column", 4)])
def test_emu_ranks_fused_gpu(plan, world):
    """the row-wise kernels fed through the fused peer data flow (world > 1) on the GPU"""
    from hugectr_b200.parallel.emu import run_ranks
    run_ranks(world, lambda c: _emu_body(plan, True, c))
