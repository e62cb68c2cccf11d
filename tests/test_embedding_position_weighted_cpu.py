"""Position-weighted inputs (DataReaderSparseParam(..., position_weighted=True)) on the CPU path: the weight gradient
dP against an fp64 autograd oracle, P = 1 against the unweighted model, emulated ranks, the rejections, the graph JSON,
the dense-file layout, exact resume, training and serving.

Error bound of dP (fp32 against the fp64 oracle).  With u = 2^-24 and gamma_n = n u / (1 - n u), a sum of n fp32
terms is within gamma_n * (sum of the terms' magnitudes) of the exact sum.  For one key occurrence the owner forms
the dot <T[key_h], g'> over ev columns (g' = g * H / W', the top gradient after the mean rescale, itself within
gamma_{H+2} of exact because W' = sum_w, or 1 when it is 0, sums H fp32 weights) and scales it by 1/H: within
gamma_{ev+H+4} of <T, g> / W' relative to sum_c |T_c g_c| / |W'|.  The requester's mean term <pooled, g> / W is
within gamma_{ev+2H+4} relative to sum_c |pooled_c g_c| / |W| (the pooled vector carries the forward's H-term sum).
The column sums add R * B of these per position in fp32, gamma_{R*B}.  So
    |dP - dP_64| <= gamma_{ev + 2H + R*B + 8} * S,   S = sum over occurrences of (sum_c |T_c g_c| + sum_c |pooled_c g_c|) / |W'|,
and the tests check this at every position, with S computed in fp64 from the oracle's operands.

The harness is shared with test_embedding_position_weighted_gpu.py."""
import json

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                               EmbeddingTableConfig)
from hugectr_b200.enums import CompressionStrategy, Optimizer_t
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

CPU = torch.device("cpu")
U = 2.0 ** -24

# lookups of the top "emb": p0 (position-weighted, table 0), u1 (unweighted one-hot, table 1), p2 (position-
# weighted, table 2); with ``shared`` a second top "emb2" reads p0 again through table 3
INPUTS = ("p0", "u1", "p2")
PW = ("p0", "p2")
HOT = {"p0": 4, "u1": 1, "p2": 8}
VOCAB = (50, 7, 300)


# ----------------------------------------------------------------------------- harness
def make_cfg(world, plan, combiner, ev=16, dynamic=None, weight_dtype="fp32", shared=False):
    """``plan``: table | row | dp; ``dynamic``: None, "grow", "admit" (threshold 2), "lru" for table 2"""
    ts = []
    for i, v in enumerate(VOCAB):
        kw = dict(weight_dtype=weight_dtype)
        if dynamic is not None and i == 2:
            kw.update(init_capacity=512)
            if dynamic == "admit":
                kw.update(admit_threshold=2)
            elif dynamic != "grow":
                kw.update(max_capacity=512, evict_strategy=dynamic)
            ts.append(EmbeddingTableConfig(str(i), -1, ev, **kw))
        else:
            ts.append(EmbeddingTableConfig(str(i), v, ev, **kw))
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, list(INPUTS), "emb", [combiner, "sum", combiner])
    names = ["0", "1", "2"]
    if shared:
        ts.append(EmbeddingTableConfig("3", VOCAB[0], ev, weight_dtype=weight_dtype))
        cfg.embedding_lookup([ts[3]], ["p0"], "emb2", ["sum"])
        names.append("3")
    if plan != "table":
        n = len(names)
        sm = [[0] * n for _ in range(world)]
        sm[0][0] = 1
        sm[world - 1][1] = 1
        for g in range(world):
            sm[g][2] = 1
        if shared:
            sm[world - 1][3] = 1
        if plan == "row":
            cfg.shard(sm, [("mp", names)])
        elif plan == "dp":
            for g in range(world):
                sm[g][0] = 1
            cfg.shard(sm, [("dp", ["0"]), ("mp", names[1:])])
        else:
            raise ValueError(plan)
    return cfg


def make_collection(dev, comm, b, plan="table", combiner="sum", pw=PW, opt=None, P=None, **kw):
    """the collection and its position weights {input: (P [1, H], grad [1, H])} (P = 1 unless given)"""
    world = comm.get_global_gpu_count() if hasattr(comm, "get_global_gpu_count") else comm.world_size
    ckw = {k: kw.pop(k) for k in ("fused", "state_dtype", "key_dtype", "act_dtype") if k in kw}
    act = ckw.pop("act_dtype", torch.float32)
    cfg = make_cfg(world, plan, combiner, **kw)
    opt = opt or CreateOptimizer(Optimizer_t.SGD)
    e = EmbeddingCollection(cfg, b, HOT, dev, act, comm, opt, seed=3, position_weighted=pw, **ckw)
    params = {n: ((P[n].clone() if P is not None else torch.ones(1, HOT[n])).to(dev).float(),
                  torch.zeros(1, HOT[n], device=dev)) for n in pw}
    e.bind_position_weights(params)
    return e, params


def make_tables(gen, ev=16, shared=False):
    t = {str(i): (torch.rand(v, ev, generator=gen, dtype=torch.float64) - 0.5) * 0.2 for i, v in enumerate(VOCAB)}
    if shared:
        t["3"] = (torch.rand(VOCAB[0], ev, generator=gen, dtype=torch.float64) - 0.5) * 0.2
    return t


def load_tables(e, tables):
    for name, w in tables.items():
        if name in e.tmap:
            e.load_table_rows(name, torch.arange(w.shape[0]), w.float())


def make_P(gen, zero_bag=False):
    """position weights in [-0.5, 1.5); with ``zero_bag`` the first two positions of p0 cancel (0.75, -0.75)"""
    P = {n: (torch.rand(1, HOT[n], generator=gen) * 2 - 0.5) for n in PW}
    if zero_bag:
        P["p0"][0, :2] = torch.tensor([0.75, -0.75])
    return P


def make_batch(gen, B, variable=True, zero_bag=False):
    """keys [B, H] per input, -1 padding in variable bags; with ``zero_bag`` sample 0 of p0 holds 2 keys"""
    keys = {}
    for i, name in enumerate(INPUTS):
        H = HOT[name]
        k = torch.randint(0, VOCAB[i], (B, H), generator=gen)
        if variable and H > 1:
            n = torch.randint(0, H + 1, (B,), generator=gen)
            n[0] = H
            if zero_bag and name == "p0":
                n[0] = 2
            k = torch.where(torch.arange(H).view(1, -1) < n.view(-1, 1), k, torch.full_like(k, -1))
        keys[name] = k
    return keys


def step(e, keys, grads, lr=0.1, rows=None):
    """one forward + backward of ``e`` on (a row window of) the batch; ``grads``: {top: [B, width]}; returns the
    outputs {top: [b, width]}"""
    dev = e.device
    for gl in e.glookups:        # (a key block per lookup: an input read twice fills two blocks)
        k = keys[gl["bottom"]] if rows is None else keys[gl["bottom"]][rows]
        e.key_slab[gl["key_off"]:gl["key_off"] + k.numel()].copy_(k.reshape(-1).to(e.key_dtype).to(dev))
    e.forward()
    outs = {t: e.top_data[t].float().cpu().clone().reshape(e.b, -1) for t in e.top_data}
    for t, g in grads.items():
        e.top_grad[t].copy_((g if rows is None else g[rows]).reshape(e.top_grad[t].shape).to(dev))
    e.backward(torch.tensor([lr], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))
    return outs


def oracle(tables, keys, P, combiner, grads, rowless=None, shared=False):
    """fp64 autograd: (outputs {top: [B, width]}, dP {input: [1, H]}, bound {input: [1, H]}) of loss =
    sum_tops <top, grad>; ``rowless``: {input: bool [B, H]} keys that read as zero vectors"""
    Pd = {n: P[n].double().clone().requires_grad_(True) for n in PW}
    ev = tables["0"].shape[1]
    S = {n: torch.zeros(1, HOT[n], dtype=torch.float64) for n in PW}
    lks = [("emb", i, name, "0" if i == 0 else str(i), combiner if name != "u1" else "sum")
           for i, name in enumerate(INPUTS)]
    if shared:
        lks.append(("emb2", 0, "p0", "3", "sum"))
    outs = {t: [] for t in grads}
    loss = 0
    for top, col, name, tab, comb in lks:
        k = keys[name]
        valid = k >= 0
        rows = tables[tab][k.clamp(min=0)]
        if rowless is not None and name in rowless:
            rows = rows * (~rowless[name]).unsqueeze(-1).double()
        w = torch.where(valid, Pd[name].expand_as(k), torch.zeros((), dtype=torch.float64)) if name in PW \
            else valid.double()
        pooled = (w.unsqueeze(-1) * rows).sum(1)
        if comb == "mean":
            sw = w.sum(1)
            Wp = torch.where(sw == 0, torch.ones_like(sw), sw)
            pooled = pooled / Wp.unsqueeze(1)
        else:
            Wp = torch.ones(k.shape[0], dtype=torch.float64)
        g = grads[top][:, col * ev:(col + 1) * ev].double() if top == "emb" else grads[top].double()
        loss = loss + (pooled * g).sum()
        outs[top].append(pooled.detach())
        if name in PW:
            t = (rows.abs() * g.abs().unsqueeze(1)).sum(-1) + (pooled.detach().abs() * g.abs()).sum(-1, keepdim=True)
            S[name] += (t * valid / Wp.detach().abs().unsqueeze(1)).sum(0, keepdim=True)
    loss.backward()
    dP = {n: Pd[n].grad.detach() for n in PW}
    return {t: torch.cat(v, 1) for t, v in outs.items()}, dP, S


def bound(S, B, R=1, ev=16):
    n = ev + 2 * max(HOT.values()) + R * B + 8
    return {k: (n * U / (1 - n * U)) * v for k, v in S.items()}


def check_dP(params, dP, S, B, R=1):
    bd = bound(S, B, R)
    for n in PW:
        got = params[n][1].double().cpu()
        err = (got - dP[n]).abs()
        assert bool((err <= bd[n] + 1e-12).all()), f"{n}: err {err.max().item()} bound {bd[n].max().item()}"


# ----------------------------------------------------------------------------- dP against the fp64 oracle
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_weight_gradient_matches_fp64_oracle(combiner):
    gen = torch.Generator().manual_seed(11)
    B = 24
    tables = make_tables(gen, shared=True)
    P = make_P(gen, zero_bag=True)
    e, params = make_collection(CPU, Comm.single(CPU), B, combiner=combiner, P=P, shared=True)
    load_tables(e, tables)
    keys = make_batch(gen, B, zero_bag=True)
    grads = {"emb": torch.randn(B, 48, generator=gen) * 0.1, "emb2": torch.randn(B, 16, generator=gen) * 0.1}
    outs = step(e, keys, grads)
    exp_out, dP, S = oracle(tables, keys, P, combiner, grads, shared=True)
    for t in outs:
        assert (outs[t].double() - exp_out[t]).abs().max().item() < 1e-5
    check_dP(params, dP, S, B)
    if combiner == "mean":
        # the W == 0 bag (sample 0 of p0: weights 0.75 and -0.75) divides by 1 and takes no mean term
        assert float(P["p0"][0, :2].sum()) == 0.0


def test_weight_gradient_with_rejected_keys_matches_fp64_oracle():
    """a dynamic table admitting keys on their second occurrence: in the second step the even positions of p2 repeat
    the first step's keys (admitted, fresh rows) and the odd ones are new (rejected: zero vectors that keep their
    place in the mean).  SGD at lr 0 keeps the rows the oracle reads."""
    gen = torch.Generator().manual_seed(5)
    B = 16
    tables = make_tables(gen)
    P = make_P(gen)
    e, params = make_collection(CPU, Comm.single(CPU), B, combiner="mean", P=P, dynamic="admit")
    load_tables(e, {n: t for n, t in tables.items() if n != "2"})
    keys = make_batch(gen, B)
    H = HOT["p2"]
    first = 1000 + torch.arange(B * H).view(B, H)
    keys["p2"] = torch.where(keys["p2"] >= 0, first, keys["p2"])
    grads = {"emb": torch.randn(B, 48, generator=gen) * 0.1}
    step(e, keys, grads, lr=0.0)
    for n in PW:
        params[n][1].zero_()
    fresh = 5000 + torch.arange(B * H).view(B, H)
    keys["p2"] = torch.where(keys["p2"] >= 0, torch.where(torch.arange(H) % 2 == 0, first, fresh), keys["p2"])
    step(e, keys, grads, lr=0.0)
    (dk, dw, _, _, _), = e.dump_table_local("2")
    t2 = torch.zeros(6000 + B * H, 16, dtype=torch.float64)
    t2[dk] = dw.double()
    rowless = {"p2": (keys["p2"] >= 0) & ~torch.isin(keys["p2"], dk)}
    assert bool(rowless["p2"].any()) and bool(((keys["p2"] >= 0) & ~rowless["p2"]).any())
    _, dP, S = oracle(dict(tables, **{"2": t2}), keys, P, "mean", grads, rowless=rowless)
    check_dP(params, dP, S, B)
    assert e.admission_stats()[("2", 0)]["rejected"] > 0


# ----------------------------------------------------------------------------- P = 1 == unweighted
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_ones_equal_unweighted_at_step_0(combiner):
    gen = torch.Generator().manual_seed(4)
    B = 16
    tables = make_tables(gen)
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-7)
    ep, _ = make_collection(CPU, Comm.single(CPU), B, combiner=combiner, opt=opt)
    eu, _ = make_collection(CPU, Comm.single(CPU), B, combiner=combiner, opt=opt, pw=())
    load_tables(ep, tables)
    load_tables(eu, tables)
    keys = make_batch(gen, B)
    grads = {"emb": torch.randn(B, 48, generator=gen) * 0.1}
    assert torch.equal(step(ep, keys, grads)["emb"], step(eu, keys, grads)["emb"])
    for gp, gu in zip(ep.groups, eu.groups):
        assert torch.equal(gp.table, gu.table) and torch.equal(gp.s0, gu.s0)


# ----------------------------------------------------------------------------- emulated ranks == one process
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("plan", ["table", "row", "dp"])
@pytest.mark.parametrize("fused", [False, True])
def test_emulated_ranks_equal_one_process(world, plan, fused):
    from hugectr_b200.parallel.emu import run_ranks
    b = 6
    B = b * world
    gen = torch.Generator().manual_seed(21)
    tables = make_tables(gen, shared=True)
    P = make_P(gen)
    keys = make_batch(gen, B)
    grads = {"emb": torch.randn(B, 48, generator=gen) * 0.1, "emb2": torch.randn(B, 16, generator=gen) * 0.1}
    _, dP, S = oracle(tables, keys, P, "mean", grads, shared=True)
    one, p1 = make_collection(CPU, Comm.single(CPU), B, combiner="mean", P=P, shared=True)
    load_tables(one, tables)
    ref = step(one, keys, grads)

    def rank_fn(comm):
        e, params = make_collection(CPU, comm, b, plan=plan, combiner="mean", P=P, shared=True, fused=fused)
        load_tables(e, tables)
        rows = slice(comm.rank * b, (comm.rank + 1) * b)
        out = step(e, keys, grads, rows=rows)
        for t in out:
            assert (out[t] - ref[t][rows]).abs().max().item() < 1e-6
        # the dense all-reduce of the partial gradients
        for n in PW:
            comm.all_reduce(params[n][1])
        check_dP(params, dP, S, B, R=world)
        for n in PW:
            assert (params[n][1] - p1[n][1]).abs().max().item() <= bound(S, B, world)[n].max().item() * 2
        return True
    assert all(run_ranks(world, rank_fn, device=CPU))


# ----------------------------------------------------------------------------- rejections and the graph JSON
def test_parameter_validation():
    P = hugectr.DataReaderSparseParam
    with pytest.raises(ValueError, match="input a"):
        P("a", 3, False, 1, position_weighted=1)
    with pytest.raises(ValueError, match="input a"):
        P("a", 3, False, 1, weighted=True, position_weighted=True)
    assert P("a", 3, False, 1, position_weighted=True).to_json()["position_weighted"] is True
    assert "position_weighted" not in P("a", 3, False, 1).to_json()


def test_collection_rejections():
    t = EmbeddingTableConfig("t", 10, 4)
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(t, "p", "top", "concat")
    with pytest.raises(ValueError, match="position-weighted input p"):
        EmbeddingCollection(cfg, 4, {"p": 2}, CPU, torch.float32, Comm.single(CPU),
                            CreateOptimizer(Optimizer_t.SGD), position_weighted={"p"})
    from hugectr_b200.parallel.emu import run_ranks
    cu = EmbeddingCollectionConfig()
    cu.embedding_lookup(t, "p", "top", "sum")
    cu.shard([[1], [1]], [("mp", ["t"])], {CompressionStrategy.Unique: ["t"]})
    cc = EmbeddingCollectionConfig()
    cc.embedding_lookup(t, "p", "top", "sum")
    cc.shard([[1], [1]], [("mp", [("t", 2)])])

    def mk(comm):
        for cfg in (cu, cc):
            with pytest.raises(ValueError, match="table t"):
                EmbeddingCollection(cfg, 4, {"p": 2}, CPU, torch.float32, comm, CreateOptimizer(Optimizer_t.SGD),
                                    position_weighted={"p"}, fused=False)
        return True
    assert all(run_ranks(2, mk, device=CPU))


def _model(reader_type=None, legacy=False, pw=True, seed=0, lr=0.05, opt=Optimizer_t.AdaGrad, batch=32,
           device=CPU, cuda_graph=False):
    solver = hugectr.CreateSolver(batchsize=batch, batchsize_eval=batch, lr=lr, vvgpu=[[0]], seed=seed,
                                  use_cuda_graph=cuda_graph)
    rp = hugectr.DataReaderParams(reader_type or hugectr.DataReaderType_t.Parquet, source=["synthetic"],
                                  eval_source="synthetic", check_type=hugectr.Check_t.Non, slot_size_array=[100, 20])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(opt), comm=Comm.single(device))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[
                            hugectr.DataReaderSparseParam("a", 3, False, 1, position_weighted=pw),
                            hugectr.DataReaderSparseParam("b", 1, True, 1)]))
    if legacy:
        m.add(hugectr.SparseEmbedding(embedding_type=hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash,
                                      workspace_size_per_gpu_in_mb=1, embedding_vec_size=8, combiner="sum",
                                      sparse_embedding_name="sa", bottom_name="a"))
        m.add(hugectr.DenseLayer(layer_type=hugectr.Layer_t.Reshape, bottom_names=["sa"], top_names=["r"],
                                 leading_dim=8))
        top = "r"
    else:
        ec = EmbeddingCollectionConfig()
        ta, tb = EmbeddingTableConfig("ta", 100, 8), EmbeddingTableConfig("tb", 20, 8)
        ec.embedding_lookup([ta, tb], ["a", "b"], "emb", ["mean", "sum"])
        m.add(ec)
        top = "emb"
    m.add(hugectr.DenseLayer(layer_type=hugectr.Layer_t.Concat, bottom_names=[top, "dense"], top_names=["x"]))
    m.add(hugectr.DenseLayer(layer_type=hugectr.Layer_t.InnerProduct, bottom_names=["x"], top_names=["y"],
                             num_output=1))
    m.add(hugectr.DenseLayer(layer_type=hugectr.Layer_t.BinaryCrossEntropyLoss, bottom_names=["y", "label"],
                             top_names=["loss"]))
    return m


def test_model_accepts_any_reader_and_rejects_legacy_tables():
    for t in (hugectr.DataReaderType_t.Norm, hugectr.DataReaderType_t.Raw):
        m = _model(reader_type=t)
        m.compile()
        assert tuple(m.position_weights["a"].shape) == (1, 3)
    with pytest.raises(ValueError, match="position-weighted input a"):
        _model(legacy=True).compile()


def test_graph_json_round_trip(tmp_path):
    from hugectr_b200.graph_json import model_to_json
    j = model_to_json(_model())
    sp = {s["top"]: s for s in j["layers"][0]["sparse"]}
    assert sp["a"]["position_weighted"] is True and "position_weighted" not in sp["b"]
    assert "position_weighted" not in json.dumps(model_to_json(_model(pw=False)))
    path = tmp_path / "g.json"
    path.write_text(json.dumps(j))
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["synthetic"], eval_source="synthetic",
                                  check_type=hugectr.Check_t.Non, slot_size_array=[100, 20])
    m2 = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m2.construct_from_json(str(path))
    prm = {p.top_name: p for p in m2.input.data_reader_sparse_param_array}
    assert prm["a"].position_weighted and not prm["b"].position_weighted


def test_onnx_export_rejects(tmp_path):
    from hugectr_b200.onnx import hugectr2onnx
    m = _model()
    m.compile()
    m.graph_to_json(str(tmp_path / "g.json"))
    with pytest.raises(ValueError, match="position-weighted input a"):
        hugectr2onnx.convert(str(tmp_path / "m.onnx"), str(tmp_path / "g.json"), str(tmp_path / "missing"))


# ----------------------------------------------------------------------------- dense files, resume
def test_dense_file_layout(tmp_path):
    """the position weights follow the network's parameters: the network's bytes are those of the model without
    the option, in the weights and in the optimizer state"""
    a, b = _model(pw=False, opt=Optimizer_t.Adam), _model(pw=True, opt=Optimizer_t.Adam)
    a.compile()
    b.compile()
    n = a.arena.num_params
    assert b.arena.num_params == n + 3 and b.arena.params[-1] is b.position_weights["a"]
    a.save_params_to_files(str(tmp_path / "a"))
    b.save_params_to_files(str(tmp_path / "b"))
    from hugectr_b200.io.checkpoint import dense_paths
    (wa, sa), (wb, sb) = dense_paths(str(tmp_path / "a"), 0), dense_paths(str(tmp_path / "b"), 0)
    ra, rb = open(wa, "rb").read(), open(wb, "rb").read()
    assert rb[:4 * n] == ra and np.array_equal(np.frombuffer(rb[4 * n:], "<f4"), np.ones(3, "<f4"))
    assert len(open(sb, "rb").read()) == len(open(sa, "rb").read()) * (n + 3) // n


def test_exact_resume(tmp_path):
    def mk():
        m = _model(seed=7, opt=Optimizer_t.Adam)
        m.compile()
        return m
    a = mk()
    pool = a.reader_train.pool
    pre = str(tmp_path / "snap")
    for i in range(6):
        a.train_on_host_batch(pool[i % len(pool)])
        if i == 2:
            a.save_params_to_files(pre, 3)
    b = mk()
    assert b.resume(pre) == 3
    for i in range(3, 6):
        b.train_on_host_batch(pool[i % len(pool)])
    assert torch.equal(a.arena.weights, b.arena.weights)
    assert not torch.equal(a.position_weights["a"].w, torch.ones(1, 3))
    for pa, pb in zip(a.ebcs_train[0].dump_table_local("ta"), b.ebcs_train[0].dump_table_local("ta")):
        assert torch.equal(pa[1], pb[1])


# ----------------------------------------------------------------------------- training and serving
def position_batches(m, n, gen):
    """batches whose label is 1 when the key at position 0 of input a is even: only position 0 carries signal"""
    from hugectr_b200.data.batch import HostBatch
    B = m.b_train
    out = []
    for _ in range(n):
        ka = torch.randint(0, 100, (B, 3), generator=gen)
        kb = torch.randint(0, 20, (B, 1), generator=gen)
        lab = (ka[:, 0] % 2 == 0).float().view(B, 1)
        dense = torch.rand(B, 2, generator=gen)
        out.append(HostBatch(lab, dense, torch.cat([ka.reshape(-1), kb.reshape(-1)]).to(m.key_dtype), None, B))
    return out


def test_training_moves_weights_toward_the_informative_position():
    gen = torch.Generator().manual_seed(3)
    m = _model(lr=0.05, opt=Optimizer_t.Adam)
    m.compile()
    # a table whose even keys point one way and odd keys the other along every column
    ta = torch.where(torch.arange(100).view(-1, 1) % 2 == 0, 0.5, -0.5) * torch.ones(100, 8)
    m.ebcs_train[0].load_table_rows("ta", torch.arange(100), ta)
    for hb in position_batches(m, 150, gen):
        m.train_on_host_batch(hb)
    P = m.position_weights["a"].w.detach().cpu().view(-1)
    # the mean pools w_0 T[k_0] + ... : the informative position gains weight over the two noise positions
    assert float(P[0]) > 1.0 and float(P[0]) > float(P[1:].max()) + 0.2, P


def test_inference_session_predicts_as_the_trained_evaluation(tmp_path):
    from hugectr_b200.inference import InferenceParams, InferenceModel
    gen = torch.Generator().manual_seed(9)
    m = _model(lr=0.05, opt=Optimizer_t.Adam)
    m.compile()
    for hb in position_batches(m, 20, gen):
        m.train_on_host_batch(hb)
    assert not torch.equal(m.position_weights["a"].w.cpu(), torch.ones(1, 3))
    pre = str(tmp_path / "m")
    m.save_params_to_files(pre)
    m.graph_to_json(str(tmp_path / "g.json"))
    m.embedding_dump(str(tmp_path / "emb"))
    from hugectr_b200.io.checkpoint import dense_paths
    sess = InferenceModel(str(tmp_path / "g.json"), InferenceParams(
        "m", 32, dense_model_file=dense_paths(pre, 0)[0], embedding_collection_path=str(tmp_path / "emb")),
        device="cpu")
    hb = position_batches(m, 1, gen)[0]
    pred = sess.predict(hb.dense.numpy(), hb.keys.numpy())
    m._load_batch(hb, False)
    for e in m.ebcs_eval:
        e.forward(False)
    m.net_eval.fprop(False)
    exp = m.net_eval.loss_layers[0].pred[:32].float().cpu().numpy()
    np.testing.assert_allclose(pred, exp, rtol=1e-6, atol=1e-7)
