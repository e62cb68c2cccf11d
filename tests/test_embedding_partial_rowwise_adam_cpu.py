"""Partial row-wise Adam for embedding-collection tables (Optimizer_t.PartialRowWiseAdam): the oracle, and
the tests that need no GPU.

Definition, for a table row r that receives gradients in a step t (the device step counter), ev columns:
  g[c]  = (sum of the row's gradient contributions, 1/nnz for mean, times the key weights) * grad_scale / scaler
  m[c]  = b1 m[c] + (1 - b1) g[c]                       per element (state 0), in the state dtype
  v[r]  = b2 v[r] + (1 - b2) (1/ev) sum_c g[c]^2        one fp32 value per row (state 1)
  w[c] -= alpha m[c] / (sqrt(v[r]) + eps),  alpha = lr sqrt(1 - b2^t) / (1 - b1^t)
m and v start at 0; rows without gradient are untouched.

The oracle below is written from that definition in fp64 on the per-row gradient sums of
test_embedding_kernels_gpu.py (oracle_reduce), not from the package's CPU path.

Error bound (stated once, used everywhere; u = 2^-24).  The kernels sum a row's n gradient rows in fp32 in
any order, so every summed column lies within e = (n + 4) u sum|g| of the exact one.  Then
  m:  |dm| <= (1 - b1) e + 4 u (b1 |m_old| + (1 - b1) |g| + |m_new|)
  S = mean_c g^2:  |dS| <= mean_c(2 |g| e + e^2) + (ev + 8) u S          (the row's fp32 sum and division)
  v:  |dv| <= (1 - b2) |dS| + 8 u (b2 v_old + (1 - b2) S)
  bias corrections: fast-math powf(b, t) is exp2(t log2 b) with approximate hardware exp2 / log2, relative
      error dp <= (t + 1) 2^-21, so 1 - b^t has relative error r_b <= b^t dp / (1 - b^t) + u, and
      alpha = lr sqrt(bc2) / bc1 relative error r_a <= r_b1 + r_b2 / 2 + 6 u
  D = sqrt(v) + eps:  |dD| <= |dv| / (2 sqrt(v)) + 4 u D,  f = alpha / D relative error r_f <= r_a + |dD| / D + 4 u
  w:  |d dw| <= f |dm| + f |m| r_f + 16 u (|dw| + |w_old| + |w_new|)
bf16 weights may additionally differ by one bf16 ulp of the new weight (stochastic rounding), and a bf16 m by
one bf16 ulp of m (round to nearest).
"""
import json
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_embedding_kernels_gpu as K  # noqa: E402
from hugectr_b200.embedding import ops as E  # noqa: E402
from hugectr_b200.enums import CompressionStrategy, Optimizer_t as O  # noqa: E402
from hugectr_b200.ops.optim import opt_reference  # noqa: E402

U = K.U
PRA = O.PartialRowWiseAdam
BF = torch.bfloat16
CPU = torch.device("cpu")
HP = dict(K.HP, epsilon=2.0 ** -10)      # beta1 0.875, beta2 0.9375
LR = K.LR


# ------------------------------------------------------------------------------------------ oracle
def prow_oracle(red, w_old, m_old, v_old, step, hp=HP, lr=LR):
    """(dw = w_new - w_old [n, ev], m_new [n, ev], v_new [n], and the bounds of the three) of the rows ``red``
    touches, in fp64 from the rows' values before the step"""
    uniq, G, A, n = red
    scaler, eps, b1, b2 = hp.get("scaler", 1.0), hp["epsilon"], hp["beta1"], hp["beta2"]
    g = G / scaler
    e = (n.view(-1, 1) + 4).double() * U * A / scaler
    m_old, v_old = m_old.double(), v_old.double()
    m = b1 * m_old + (1 - b1) * g
    S = (g * g).mean(1)
    v = b2 * v_old + (1 - b2) * S
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    alpha = lr * math.sqrt(bc2) / bc1
    D = v.sqrt() + eps
    f = alpha / D
    dw = -f.view(-1, 1) * m
    tm = (1 - b1) * e + 4 * U * (b1 * m_old.abs() + (1 - b1) * g.abs() + m.abs())
    dS = (2 * g.abs() * e + e * e).mean(1) + (g.shape[1] + 8) * U * S
    tv = (1 - b2) * dS + 8 * U * (b2 * v_old.abs() + (1 - b2) * S)
    dp = (step + 1) * 2.0 ** -21
    ra = (b1 ** step * dp / bc1 + U) + (b2 ** step * dp / bc2 + U) / 2 + 6 * U
    dD = tv / (2 * v.sqrt().clamp(min=1e-300)) + 4 * U * D
    rf = ra + dD / D + 4 * U
    tw = f.view(-1, 1) * tm + (f * rf).view(-1, 1) * m.abs() \
        + 16 * U * (dw.abs() + w_old.double().abs() + (w_old.double() + dw).abs())
    return dw, m, v, tw, tm, tv


def check_prow(what, case, tab, m, v, new, step, hp=HP, lr=LR, grad_scale=1.0, bf16=False):
    """result ``new`` = (w, m, v) against the oracle; rows no pair touches must not change"""
    P = case.pitch
    red = K.oracle_reduce(case, grad_scale)
    check_red(what, red, P, tab, m, v, new, step, hp, lr, bf16)


def check_red(what, red, P, tab, m, v, new, step, hp=HP, lr=LR, bf16=False):
    uniq = red[0]
    w_old = tab.view(-1, P)[uniq].double()
    dw, m_ref, v_ref, tw, tm, tv = prow_oracle(red, w_old, m.view(-1, P)[uniq], v[uniq], step, hp, lr)
    w_new, m_new, v_new = (x.cpu() for x in new)
    assert v_new.dtype == torch.float32 and v_new.numel() == v.numel()
    if bf16:
        tw = tw + K.bf16_ulp(w_old + dw)
    K.assert_close_bound(f"{what} dw", w_new.view(-1, P)[uniq].double() - w_old, dw, tw)
    K.assert_close_bound(f"{what} m", m_new.view(-1, P)[uniq], m_ref, tm, bf16=m_new.dtype == BF)
    K.assert_close_bound(f"{what} v", v_new[uniq], v_ref, tv)
    keep = torch.ones(tab.numel() // P, dtype=torch.bool)
    keep[uniq] = False
    assert torch.equal(w_new.view(-1, P)[keep], tab.view(-1, P)[keep]), f"{what}: untouched w rows changed"
    assert torch.equal(m_new.view(-1, P)[keep], m.view(-1, P)[keep]), f"{what}: untouched m rows changed"
    assert torch.equal(v_new[keep], v[keep]), f"{what}: untouched v rows changed"


def init_prow(rows, pitch, gen, wdt=torch.float32, mdt=torch.float32):
    """weights, first moments (rounded to their dtype) and fp32 second moments as after some training"""
    tab = (torch.randn(rows * pitch, generator=gen) * 0.1).to(wdt)
    m = (torch.randn(rows * pitch, generator=gen) * 0.01).to(mdt)
    v = torch.rand(rows, generator=gen) * 1e-2 + 1e-4
    return tab, m, v


# ------------------------------------------------------------------------------------------ oracle vs CPU paths
def test_oracle_matches_package_cpu_paths_over_steps():
    """opt_reference, update_rows (the CPU path of backward_accum + update) on a case with every lookup
    feature, loss scaler and grad_scale != 1, five steps t = 1..5 from the previous step's state"""
    gen = torch.Generator().manual_seed(1)
    case = K.features_case(8, torch.float32, gen, batch=40)
    tab, m, v = init_prow(case.rows, case.pitch, gen)
    m.zero_()
    v.zero_()
    hp = dict(HP, scaler=4.0)
    for t in range(1, 6):
        tt, mm, vv = tab.clone(), m.clone(), v.clone()
        ws = E.UniqueWorkspace(case.pairs, case.pitch, CPU)
        E.backward_accum(case.lookups, None, tt, case.pitch, case.keys, case.grads, case.batch, ws, 0.5,
                         nnz_bufs=case.nnz)
        E.update(PRA, tt, mm, vv, case.pitch, ws, hp, torch.tensor([LR]), torch.tensor([t], dtype=torch.int32))
        check_prow(f"update_rows t={t}", case, tab, m, v, (tt, mm, vv), t, hp=hp, grad_scale=0.5)
        # opt_reference on the fp32-rounded sums of the same rows
        uniq, G, A, n = red = K.oracle_reduce(case, 0.5)
        w2, m2, v2 = tab.view(-1, 8)[uniq].clone(), m.view(-1, 8)[uniq].clone(), v[uniq].clone()
        opt_reference(PRA, w2, m2, v2, G.float(), hp, LR, t)
        dw, m_ref, v_ref, tw, tm, tv = prow_oracle(red, tab.view(-1, 8)[uniq], m.view(-1, 8)[uniq], v[uniq], t, hp)
        K.assert_close_bound(f"opt_reference t={t} dw", w2.double() - tab.view(-1, 8)[uniq].double(), dw, tw)
        K.assert_close_bound(f"opt_reference t={t} m", m2, m_ref, tm)
        K.assert_close_bound(f"opt_reference t={t} v", v2, v_ref, tv)
        tab, m, v = tt, mm, vv


def _wrong(case, tab, m, v, step, variant):
    """fp32 results (w, m, v) of a wrong rule"""
    P = case.pitch
    uniq, G, _, n = K.oracle_reduce(case)
    b1, b2, eps = HP["beta1"], HP["beta2"], HP["epsilon"]
    w, mm, vv = tab.clone().view(-1, P), m.clone().view(-1, P), v.clone()
    m0, v0, g = m.view(-1, P)[uniq].double(), v[uniq].double().view(-1, 1), G
    mn = b1 * m0 + (1 - b1) * g
    t = step - 1 if variant == "t-1" else step
    alpha = LR * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    if variant == "sum":
        vn = b2 * v0 + (1 - b2) * (g * g).sum(1, keepdim=True)
    elif variant == "elementwise":
        vn = b2 * v0 + (1 - b2) * g * g
    elif variant == "partial":       # v from the row's first contribution only
        keys = case.keys[0].view(case.batch, -1)
        first = torch.stack([case.grads[0].view(case.batch, P)[(keys == r).any(1).nonzero()[0, 0]].double()
                             for r in uniq])
        vn = b2 * v0 + (1 - b2) * (first * first).mean(1, keepdim=True)
    else:
        vn = b2 * v0 + (1 - b2) * (g * g).mean(1, keepdim=True)
    mw = m0 if variant == "old-m" else mn
    w[uniq] = (w[uniq].double() - alpha * mw / (vn.sqrt() + eps)).float()
    mm[uniq] = mn.float()
    vv[uniq] = vn.mean(1).float()
    return w.view(-1), mm.view(-1), vv


def test_oracle_rejects_wrong_rules():
    gen = torch.Generator().manual_seed(2)
    case = K.single_case(K.class_keys(512, 8, 3000, gen), 512, 8, 16, 3000, torch.float32, gen)
    tab, m, v = init_prow(3000, 16, gen)
    step = 3
    check_prow("exact", case, tab, m, v, _wrong(case, tab, m, v, step, "none"), step)
    for variant in ("sum", "elementwise", "partial", "t-1", "old-m"):
        with pytest.raises(AssertionError, match="outside the bound"):
            check_prow(variant, case, tab, m, v, _wrong(case, tab, m, v, step, variant), step)


@pytest.mark.parametrize("step", [1, 4])
def test_equal_magnitude_rows_follow_elementwise_adam(step):
    """a row whose |g[c]| is the same in every column, from v equal in every column, follows element-wise
    Adam (opt_reference) within the bound"""
    gen = torch.Generator().manual_seed(step)
    n, ev = 64, 24
    a = torch.rand(n, 1, generator=gen) * 0.1 + 0.01
    sign = torch.randint(0, 2, (n, ev), generator=gen).float() * 2 - 1
    G = (a * sign).double()
    w = torch.randn(n, ev, generator=gen) * 0.1
    m = torch.randn(n, ev, generator=gen) * 0.01
    v = torch.rand(n, generator=gen) * 1e-2
    wa, ma, va = w.clone(), m.clone(), v.view(-1, 1).expand(n, ev).contiguous()
    opt_reference(O.Adam, wa, ma, va, G.float(), HP, LR, step)
    red = (torch.arange(n), G, G.abs(), torch.ones(n, dtype=torch.long))
    dw, m_ref, v_ref, tw, tm, tv = prow_oracle(red, w, m, v, step)
    K.assert_close_bound("adam dw", wa.double() - w.double(), dw, tw)
    K.assert_close_bound("adam m", ma, m_ref, tm)
    K.assert_close_bound("adam v", va, v_ref.view(-1, 1).expand(n, ev), tv.view(-1, 1).expand(n, ev))


# ------------------------------------------------------------------------------------------ API
def test_partial_rowwise_adam_is_rejected_outside_embedding_collections():
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.sok import OptimizerWrapper
    o = hugectr.CreateOptimizer(PRA, beta1=0.8, beta2=0.99, epsilon=1e-8)
    solver = hugectr.CreateSolver(batchsize=8, batchsize_eval=8, vvgpu=[[0]], use_embedding_collection=True)
    reader = hugectr.DataReaderParams(data_reader_type=hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.1"],
                                      eval_source="synthetic:1.1", check_type=hugectr.Check_t.Non, slot_size_array=[10])
    with pytest.raises(ValueError, match=r"PartialRowWiseAdam.*EmbeddingTableConfig\(opt_params=...\)"):
        hugectr.Model(solver, reader, o, comm=Comm.single(CPU))
    with pytest.raises(ValueError, match=r"PartialRowWiseAdam.*EmbeddingTableConfig\(opt_params=...\)"):
        hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 1, 8, "sum", "e", "d",
                                [10], optimizer=o)
    with pytest.raises(ValueError, match=r"PartialRowWiseAdam.*EmbeddingTableConfig\(opt_params=...\)"):
        OptimizerWrapper(PRA)
    assert O.PartialRowWiseAdam.value == 8 and O.RowWiseAdaGrad.value == 7
    assert E.OPT_CODE[PRA] == 8


def test_graph_json_of_the_optimizer_round_trips():
    from hugectr_b200.solver import CreateOptimizer, OptParamsPy
    o = CreateOptimizer(PRA, beta1=0.8, beta2=0.99, epsilon=1e-6)
    j = o.to_json()
    assert j["type"] == "PartialRowWiseAdam" and j["adam_hparam"] == {"beta1": 0.8, "beta2": 0.99, "epsilon": 1e-6}
    b = OptParamsPy.from_json(json.loads(json.dumps(j)))
    assert (b.optimizer_type, b.beta1, b.beta2, b.epsilon) == (PRA, 0.8, 0.99, 1e-6)


def test_dlrm_builder_gives_every_table_the_optimizer():
    from hugectr_b200.models.dlrm import build_dlrm_dcnv2
    from hugectr_b200.parallel.comm import Comm
    m = build_dlrm_dcnv2(batchsize=32, num_gpus=1, table_sizes=[50, 30], multi_hot=[2, 1], ev_size=16,
                         bottom=(16, 16), top=(16, 1), projection_dim=16, cross_layers=1, mixed=False,
                         embedding_optimizer="partial_rowwise_adam", comm=Comm.single(CPU))
    tables = m.ebc_configs[0].tables()
    assert all(t.opt_params.optimizer_type == PRA and (t.opt_params.beta1, t.opt_params.beta2, t.opt_params.epsilon)
               == (0.9, 0.999, 1e-7) for t in tables)
    assert m.opt_params.optimizer_type == O.AdaGrad
    with pytest.raises(ValueError, match="embedding_optimizer"):
        build_dlrm_dcnv2(batchsize=32, num_gpus=1, table_sizes=[50], multi_hot=[1], embedding_optimizer="adamw",
                         comm=Comm.single(CPU))


def test_planner_accounts_for_the_layout():
    """m per weight (state_bytes 4 or 2) and v per row (state_row_bytes 4)"""
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES
    from hugectr_b200.tools.planner import plan_tables
    rows = sum(CRITEO_TB_TABLE_SIZES)
    for wb, sb in ((4, 4), (2, 2)):
        gb = plan_tables(CRITEO_TB_TABLE_SIZES, CRITEO_TB_MULTI_HOT, 128, 1, weight_bytes=wb, state_bytes=sb,
                         state_row_bytes=4)[2]["memory_gb"][0]
        assert gb == pytest.approx(rows * (128 * (wb + sb) + 4) / 1e9)


# ------------------------------------------------------------------------------------------ collections
def _opt(b1=0.875, b2=0.9375, eps=2.0 ** -10):
    from hugectr_b200.solver import CreateOptimizer
    return CreateOptimizer(PRA, beta1=b1, beta2=b2, epsilon=eps)


def _mixed_collection(dev, state_dtype=torch.float32):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.solver import CreateOptimizer
    cfg = EmbeddingCollectionConfig()
    ts = [EmbeddingTableConfig("pa", 100, 16, opt_params=_opt()),
          EmbeddingTableConfig("adam", 80, 16, opt_params=CreateOptimizer(O.Adam, beta1=0.875, beta2=0.9375)),
          EmbeddingTableConfig("rw", 60, 16, opt_params=CreateOptimizer(O.RowWiseAdaGrad, initial_accu_value=0.1)),
          EmbeddingTableConfig("pb", 70, 16, opt_params=_opt(0.8, 0.99)),
          EmbeddingTableConfig("padp", 40, 16, opt_params=_opt())]
    cfg.embedding_lookup(ts, ["d0", "d1", "d2", "d3", "d4"], "emb", ["sum", "mean", "sum", "sum", "sum"])
    cfg.shard([[1, 1, 1, 1, 1]], [("mp", ["pa", "adam", "rw", "pb"]), ("dp", ["padp"])])
    return EmbeddingCollection(cfg, 16, {"d0": 3, "d1": 2, "d2": 1, "d3": 2, "d4": 2}, dev, torch.float32,
                               Comm.single(dev), CreateOptimizer(O.SGD), seed=1, state_dtype=state_dtype)


HOT = ((100, 3), (80, 2), (60, 1), (70, 2), (40, 2))


def _batch(e, gen):
    keys = torch.cat([torch.randint(0, v, (16 * h,), generator=gen) for v, h in HOT]).int()
    return keys, torch.randn(e.top_grad["emb"].shape, generator=gen) * 0.1


def _step(e, keys, grad, lr, st):
    e.set_keys(keys.to(e.device))
    e.forward()
    e.top_grad["emb"].copy_(grad.to(e.device))
    e.backward(lr, st)


def _table_red(keys, grad, ti, ev=16):
    """(uniq, G, A, n) of table ti (sum combiner) of a _mixed_collection batch"""
    off = sum(16 * h for _, h in HOT[:ti])
    h = HOT[ti][1]
    rows = keys[off:off + 16 * h].long()
    g = grad[:, ti * ev:(ti + 1) * ev].double().repeat_interleave(h, 0)
    uniq, inv = torch.unique(rows, return_inverse=True)
    G = torch.zeros(uniq.numel(), ev, dtype=torch.float64).index_add_(0, inv, g)
    A = torch.zeros_like(G).index_add_(0, inv, g.abs())
    return uniq, G, A, torch.bincount(inv)


def _slice_state(e, name):
    """(group, table slice, w view, m view, v view) of table ``name``"""
    for g in e.groups:
        for sl in g.table_slices:
            if sl["table"] == name:
                lo, hi = sl["row_off"], sl["row_off"] + sl["rows"]
                return g, g.table.view(-1, g.pitch)[lo:hi], g.s0.view(-1, g.pitch)[lo:hi], g.s1[lo:hi]


def test_groups_keep_their_own_optimizer_and_hyper_parameters():
    e = _mixed_collection(CPU)
    by = {sl["table"]: g for g in e.groups for sl in g.table_slices}
    assert len({id(g) for g in by.values()}) == 5
    assert by["pa"].opt.optimizer_type == PRA and by["pa"].prow_adam and not by["pa"].rowwise
    assert by["pb"].opt.beta1 == 0.8 and [s["table"] for s in by["pb"].table_slices] == ["pb"]
    assert by["adam"].opt.optimizer_type == O.Adam and by["rw"].opt.optimizer_type == O.RowWiseAdaGrad
    assert by["padp"].kind == "dp" and by["padp"].prow_adam


def test_collection_cpu_path_follows_the_oracle_over_steps():
    """every partial row-wise Adam table (model- and data-parallel, two sets of betas) against the oracle for
    t = 1..5, beside Adam and row-wise AdaGrad tables of the same width"""
    e = _mixed_collection(CPU)
    gen = torch.Generator().manual_seed(0)
    lr = torch.tensor([LR])
    for t in range(1, 6):
        keys, grad = _batch(e, gen)
        before = {n: [x.clone() for x in _slice_state(e, n)[1:]] for n in ("pa", "pb", "padp")}
        adam_m = _slice_state(e, "adam")[2].clone()
        _step(e, keys, grad, lr, torch.tensor([t], dtype=torch.int32))
        for n, ti in (("pa", 0), ("pb", 3), ("padp", 4)):
            g, w, m, v = _slice_state(e, n)
            hp = dict(beta1=g.opt.beta1, beta2=g.opt.beta2, epsilon=g.opt.epsilon)
            red = _table_red(keys, grad, ti)
            if g.kind == "dp":    # an all-reduced dense gradient: summed in another order
                red = (red[0], red[1], red[2], red[3] + 16)
            check_red(f"{n} t={t}", red, 16, before[n][0].reshape(-1), before[n][1].reshape(-1), before[n][2],
                      (w.reshape(-1), m.reshape(-1), v), t, hp=hp)
        assert not torch.equal(adam_m, _slice_state(e, "adam")[2])   # Adam trains with its per-element rule


@pytest.mark.parametrize("sdt", [torch.float32, BF])
def test_state_layout_and_memory(sdt):
    """s0 = m: [rows * pitch] in the state dtype; s1 = v: [rows] fp32 with bf16 state too; both zero"""
    e = _mixed_collection(CPU, state_dtype=sdt)
    for g in e.groups:
        if not g.prow_adam:
            continue
        mdt = sdt if g.kind == "mp" else torch.float32
        assert g.s0.dtype == mdt and g.s0.numel() == g.rows * g.pitch and not bool(g.s0.any())
        assert g.s1.dtype == torch.float32 and g.s1.shape == (g.rows,) and not bool(g.s1.any())
        assert g.state_pitches == (g.pitch, 1)
    assert e.memory_bytes() == sum(t.numel() * t.element_size() for g in e.groups
                                   for t in (g.table, g.s0, g.s1) if t is not None)


# ------------------------------------------------------------------------------------------ model
def tiny_model(wdt, seed=7, dyn=False, table_opt="prow", dev=CPU, graph=False):
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    sizes, hot = [50, 40, 30, 20], [2, 1, 1, 2]
    solver = hugectr.CreateSolver(model_name="prow", seed=seed, batchsize=32, batchsize_eval=32,
                                  vvgpu=[[0]], lr=0.05, use_mixed_precision=False, use_cuda_graph=graph,
                                  use_embedding_collection=True, warmup_steps=1, max_eval_batches=1)
    reader = hugectr.DataReaderParams(
        data_reader_type=hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.1"], eval_source="synthetic:1.1",
        check_type=hugectr.Check_t.Non, slot_size_array=sizes,
        async_param=hugectr.AsyncParam(1, 16, shuffle=False, multi_hot_reader=True, is_dense_float=True))
    opt = hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, hugectr.Update_t.Global, initial_accu_value=0.0,
                                  epsilon=1e-8)
    m = hugectr.Model(solver, reader, opt, comm=Comm.single(dev))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=13, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam(f"data{i}", hot[i], True, 1)
                                                        for i in range(4)]))
    to = _opt(0.9, 0.999, 1e-8) if table_opt == "prow" else hugectr.CreateOptimizer(O.Adam, epsilon=1e-8)
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
def test_model_trains_round_trips_and_resumes(tmp_path, wdt, dyn):
    a = tiny_model(wdt, dyn=dyn)
    e = a.ebcs_train[0]
    assert all(g.prow_adam for g in e.groups) and sorted(g.kind for g in e.groups) == ["dp", "mp"]
    pool = a.reader_train.pool
    t0 = [g.table.clone() for g in e.groups]
    pre = str(tmp_path / "snap")
    losses = []
    for i in range(7):
        a.train_on_host_batch(pool[i % len(pool)])
        losses.append(a.get_current_loss())
        if i == 4:
            a.save_params_to_files(pre, 5)
    assert all(math.isfinite(x) for x in losses)
    for g, t in zip(e.groups, t0):
        assert not torch.equal(t, g.table) and bool(g.s0.any()) and bool((g.s1 > 0).any()), g.kind
    if dyn:   # more distinct keys than the 16 initial rows: the model grew the dynamic table
        assert any(sl["rows"] > 16 for g in e.groups for sl in g.table_slices if sl["dynamic"])
        assert all(g.s1.numel() == g.rows and g.s0.numel() == g.rows * g.pitch for g in e.groups)
    assert e.memory_bytes() == sum(g.table.numel() * g.table.element_size() + 4 * g.rows * (g.pitch + 1)
                                   for g in e.groups)
    # graph JSON
    a.graph_to_json(str(tmp_path / "g.json"))
    tj = [l for l in json.load(open(tmp_path / "g.json"))["layers"] if l["type"] == "EmbeddingCollection"][0]
    assert all(t["optimizer"]["type"] == "PartialRowWiseAdam" and t["optimizer"]["adam_hparam"]["beta2"] == 0.999
               for t in tj["tables"])
    import hugectr_b200 as hugectr
    from hugectr_b200.parallel.comm import Comm
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]],
                                  use_embedding_collection=True, use_cuda_graph=False)
    m2 = hugectr.Model(solver, a.reader_params, a.opt_params, comm=Comm.single(CPU))
    m2.construct_from_json(str(tmp_path / "g.json"))
    assert all(t.opt_params.optimizer_type == PRA and t.opt_params.epsilon == 1e-8
               for t in m2.ebc_configs[0].tables())
    # dump -> load -> dump is byte-identical, both states included
    d1 = {str(i): e.dump_table_local(str(i)) for i in range(4)}
    b = tiny_model(wdt, seed=99, dyn=dyn)
    for name, parts in d1.items():
        for keys, w, col0, sts, kind in parts:
            assert len(sts) == 2 and sts[0].shape == w.shape and sts[1].shape == w.shape
            assert torch.equal(sts[1], sts[1][:, :1].expand_as(sts[1]))      # v broadcast over the columns
            b.ebcs_train[0].load_table_rows(name, keys, w, sts)
    for name, parts in d1.items():
        for x, y in zip(parts, b.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(x[0], y[0])
            for j in (1,):
                assert x[j].numpy().tobytes() == y[j].numpy().tobytes()
            for s in (0, 1):
                assert x[3][s].numpy().tobytes() == y[3][s].numpy().tobytes()
    if not dyn:
        # resume from the step-5 snapshot: bit-identical continuation (see the row-wise AdaGrad test for why a
        # dynamic table does not resume bit-identically with any optimizer)
        c = tiny_model(wdt)
        assert c.resume(pre) == 5
        for i in range(5, 7):
            c.train_on_host_batch(pool[i % len(pool)])
        assert float((a.arena.weights - c.arena.weights).abs().max()) == 0.0
        for name in d1:
            for pa, pc in zip(e.dump_table_local(name), c.ebcs_train[0].dump_table_local(name)):
                assert torch.equal(pa[1], pc[1]) and torch.equal(pa[3][0], pc[3][0]) and torch.equal(pa[3][1], pc[3][1])


def test_adam_checkpoints_convert_both_ways(tmp_path):
    """an Adam checkpoint loads with m as it is and v as the row mean of Adam's second moments; a partial
    row-wise checkpoint loads into Adam tables with every element of v holding its row's value"""
    ada = tiny_model("fp32", table_opt="adam")
    for i in range(3):
        ada.train_on_host_batch(ada.reader_train.pool[i])
    pre = str(tmp_path / "adam")
    ada.save_params_to_files(pre, 3)
    pr = tiny_model("fp32", seed=5)
    pr.embedding_load(pre + "_ebc_3")
    for name in ("0", "1", "2", "3"):
        for pa, pp in zip(ada.ebcs_train[0].dump_table_local(name), pr.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pa[1], pp[1]) and torch.equal(pa[3][0], pp[3][0])
            assert torch.equal(pp[3][1], pa[3][1].double().mean(1, keepdim=True).float().expand_as(pa[3][1]))
    pr.save_params_to_files(pre + "pr", 3)
    back = tiny_model("fp32", seed=6, table_opt="adam")
    back.embedding_load(pre + "pr_ebc_3")
    for name in ("0", "1", "2", "3"):
        for pp, pb in zip(pr.ebcs_train[0].dump_table_local(name), back.ebcs_train[0].dump_table_local(name)):
            assert torch.equal(pp[3][0], pb[3][0]) and torch.equal(pp[3][1], pb[3][1])


# ------------------------------------------------------------------------------------------ eviction
def evicting_collection(dev, opt, sdt=torch.float32):
    """one evicting table (64 ways) with optimizer ``opt``"""
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.parallel.comm import Comm
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig("t", -1, 8, init_capacity=64, max_capacity=64, evict_strategy="lru",
                                               opt_params=opt)], ["k"], "emb", ["sum"])
    return EmbeddingCollection(cfg, 4, {"k": 2}, dev, torch.float32, Comm.single(dev), opt, seed=3,
                               key_dtype=torch.int64, state_dtype=sdt)


def admit_with_stale_state(e):
    """fills every state with stale values, admits 20 keys through a checkpoint load without state; returns
    (the admitted keys' arena rows, the group)"""
    g = e.groups[0]
    for s in (g.s0, g.s1):
        if s is not None:
            s.fill_(0.375)
    keys = torch.arange(100, 120, dtype=torch.int64) * 7919
    e.load_table_rows("t", keys, torch.ones(20, 8))
    dk, dr = e._dyn_hash("t", g.table_slices[0]).dump()
    assert torch.equal(dk, keys)
    return (dr + g.table_slices[0]["row_off"]).to(g.s0.device), g


def test_evicting_table_admits_ways_with_zero_moments_cpu():
    e = evicting_collection(CPU, _opt())
    rows, g = admit_with_stale_state(e)
    assert not bool(g.s0.view(-1, 8)[rows].any()) and not bool(g.s1[rows].any())
    keep = torch.ones(g.rows, dtype=torch.bool)
    keep[rows] = False
    assert bool((g.s0.view(-1, 8)[keep] == 0.375).all()) and bool((g.s1[keep] == 0.375).all())


# ------------------------------------------------------------------------------------------ emulated ranks
def _make_cfg(world, plan, unique):
    from hugectr_b200.embedding.collection import EmbeddingCollectionConfig, EmbeddingTableConfig
    sizes = [1000, 37, 5000, 64, 3000]
    hot = {"d0": 3, "d1": 1, "d2": 12, "d3": 2, "d4": 4}
    ts = [EmbeddingTableConfig(str(i), sizes[i], 16) for i in range(5)]
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, list(hot), "emb", ["sum", "mean", "sum", "sum", "mean"])
    extra = [{CompressionStrategy.Unique: ["0", "2", "4"]}] if unique else []
    if plan == "mixed":
        sm = [[0] * 5 for _ in range(world)]
        for g in range(world):
            sm[g][2] = 1            # table 2 row-sharded over all ranks
            sm[g][3] = 1            # table 3 data parallel
        sm[0][0] = 1
        sm[world - 1][1] = 1
        sm[world // 2][4] = 1
        cfg.shard(sm, [("mp", ["0", "1", "2", "4"]), ("dp", ["3"])], *extra)
    elif plan == "column":
        cfg.shard([[1] * 5 for _ in range(world)], [("mp", ["0", "1", ("2", world), "3", "4"])])
    return cfg, sizes, hot


def emu_body(plan, fused, unique, c):
    """one collection per emulated rank with partial row-wise Adam on every table, three steps (t = 1..3)
    against one process holding the whole batch.  Table-wise, row-sharded and data-parallel tables equal
    the single process (weights and both moments); a column-split table keeps one v per column slice, so
    each slice is checked against the oracle applied with the slice's own width (one step)"""
    from hugectr_b200.embedding.collection import EmbeddingCollection
    from hugectr_b200.parallel.comm import Comm
    world, rank, dev = c.world_size, c.rank, c.device
    b, ev = 32, 16
    cfg, sizes, hot = _make_cfg(world, plan, unique)
    opt = _opt(0.875, 0.9375, 1e-6)
    e = EmbeddingCollection(cfg, b, hot, dev, torch.float32, c, opt, seed=1, fused=fused)
    assert all(g.prow_adam for g in e.groups)
    ref = EmbeddingCollection(_make_cfg(1, "none", False)[0], b * world, hot, CPU, torch.float32, Comm.single(CPU),
                              opt, seed=1)
    gen = torch.Generator().manual_seed(5)
    full = {str(i): torch.randn(sizes[i], ev, generator=gen) * 0.1 for i in range(5)}
    for n, w in full.items():
        k = torch.arange(w.shape[0])
        e.load_table_rows(n, k, w)
        ref.load_table_rows(n, k, w)
    lr = torch.tensor([0.05])
    split = {n for n in full if e.placement[n].col_factor > 1}
    steps = 1 if split else 3
    for it in range(steps):
        st = torch.tensor([it + 1], dtype=torch.int32)
        gk = [torch.randint(0, sizes[i], (b * world, h), generator=gen) for i, h in enumerate(hot.values())]
        grad = torch.randn(b * world, 5 * ev, generator=gen) * 0.1
        e.set_keys(torch.cat([k[rank * b:(rank + 1) * b].reshape(-1) for k in gk]).int().to(dev))
        ref.set_keys(torch.cat([k.reshape(-1) for k in gk]).int())
        e.forward(); ref.forward()
        e.top_grad["emb"].copy_(grad[rank * b:(rank + 1) * b].to(dev))
        ref.top_grad["emb"].copy_(grad)
        e.backward(lr.to(dev), st.to(dev)); ref.backward(lr, st)
        if dev.type == "cuda":
            torch.cuda.synchronize()
        c.barrier()
    for n in full:
        rk, rw, _, rs, _ = ref.dump_table_local(n)[0]
        for (k, w, c0, sts, kind) in e.dump_table_local(n):
            wd = w.shape[1]
            if n not in split:
                assert (w - rw[k][:, c0:c0 + wd]).abs().max().item() < 2e-4, f"rank {rank} table {n} w"
                torch.testing.assert_close(sts[0], rs[0][k][:, c0:c0 + wd], rtol=1e-4, atol=1e-7)
                torch.testing.assert_close(sts[1], rs[1][k][:, c0:c0 + wd], rtol=1e-4, atol=1e-9)
                continue
            ti = int(n)
            rows = gk[ti].reshape(-1)
            g = grad[:, ti * ev + c0:ti * ev + c0 + wd].double().repeat_interleave(hot[f"d{ti}"], 0)
            uniq, inv = torch.unique(rows, return_inverse=True)
            G = torch.zeros(uniq.numel(), wd, dtype=torch.float64).index_add_(0, inv, g)
            A = torch.zeros_like(G).index_add_(0, inv, g.abs())
            w0 = full[n][:, c0:c0 + wd]
            dw, m_ref, v_ref, tw, tm, tv = prow_oracle((uniq, G, A, torch.bincount(inv)), w0[uniq],
                                                       torch.zeros(uniq.numel(), wd), torch.zeros(uniq.numel()), 1,
                                                       dict(beta1=0.875, beta2=0.9375, epsilon=1e-6), 0.05)
            pos = torch.searchsorted(k, uniq)
            K.assert_close_bound(f"rank {rank} slice {c0} dw", w[pos].double() - w0[uniq].double(), dw, tw)
            K.assert_close_bound(f"rank {rank} slice {c0} v", sts[1][pos, 0], v_ref, tv)
            # and the slice's own v differs from the unsplit table's
            assert not torch.allclose(sts[1][pos, 0], rs[1][uniq, 0], rtol=1e-3)
    c.barrier()


@pytest.mark.parametrize("plan,world,fused,unique", [("mixed", 2, False, False), ("mixed", 4, False, False),
                                                     ("mixed", 2, True, False), ("mixed", 4, True, False),
                                                     ("mixed", 2, False, True), ("mixed", 4, False, True),
                                                     ("column", 2, False, False)])
def test_emu_ranks_equal_one_process_cpu(plan, world, fused, unique):
    """2 and 4 emulated ranks on the CPU, on the collective path, with the fused (peer-store) data flow
    forced and with the Unique exchange: table-wise, row-sharded and data-parallel plans equal one process;
    a column factor of 2 matches the oracle per column slice"""
    from hugectr_b200.parallel.emu import run_ranks
    run_ranks(world, lambda c: emu_body(plan, fused, unique, c), device=CPU,
              p2p="force" if fused else (False if unique else True))
