"""Weighted embedding-collection lookups (DataReaderSparseParam(..., weighted=True)) on the CPU path: an fp64
oracle written from the semantics in docs/embedding.md, emulated ranks over every placement, the all-ones
invariant, the rejections, the graph JSON, the readers and a small weighted model.

The harness (``make_collection`` / ``make_batch`` / ``oracle_*``) is shared with test_embedding_weighted_gpu.py."""
import json
import os

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

# three inputs: two weighted multi-hot ones around an unweighted one-hot one
INPUTS = ("w0", "u1", "w2")
WEIGHTED = ("w0", "w2")


# ----------------------------------------------------------------------------- harness
def make_cfg(world, plan, combiner, ev=16, vocab=(50, 7, 300), dynamic=None, weight_dtype="fp32"):
    """one batch-major top "emb" over three tables; ``plan``: table | row | column | dp (world > 1)"""
    ts = []
    for i, v in enumerate(vocab):
        kw = dict(weight_dtype=weight_dtype)
        if dynamic is not None and i == 2:
            kw.update(init_capacity=512)
            if dynamic != "grow":
                kw.update(max_capacity=512, evict_strategy=dynamic)
            ts.append(EmbeddingTableConfig(str(i), -1, ev, **kw))
        else:
            ts.append(EmbeddingTableConfig(str(i), v, ev, **kw))
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, list(INPUTS), "emb", [combiner, "sum", combiner])
    if plan != "table":
        sm = [[0] * 3 for _ in range(world)]
        sm[0][0] = 1
        sm[world - 1][1] = 1
        for g in range(world):
            sm[g][2] = 1
        if plan == "row":
            cfg.shard(sm, [("mp", ["0", "1", "2"])])
        elif plan == "column":
            for g in range(world):
                sm[g][0] = 1
            cfg.shard(sm, [("mp", [("0", world), "1", "2"])])
        elif plan == "dp":
            for g in range(world):
                sm[g][0] = 1
            cfg.shard(sm, [("dp", ["0"]), ("mp", ["1", "2"])])
        else:
            raise ValueError(plan)
    return cfg


def make_collection(dev, comm, b, hot, plan="table", combiner="sum", weighted=WEIGHTED, opt=None, **kw):
    world = comm.get_global_gpu_count() if hasattr(comm, "get_global_gpu_count") else comm.world_size
    ckw = {k: kw.pop(k) for k in ("fused", "state_dtype", "key_dtype") if k in kw}
    cfg = make_cfg(world, plan, combiner, **kw)
    opt = opt or CreateOptimizer(Optimizer_t.SGD)
    return EmbeddingCollection(cfg, b, hot, dev, torch.float32, comm, opt, seed=3, weighted=weighted, **ckw)


def load_tables(e, tables):
    for name, w in tables.items():
        e.load_table_rows(name, torch.arange(w.shape[0]), w.float())


def make_tables(gen, vocab=(50, 7, 300), ev=16):
    return {str(i): (torch.rand(v, ev, generator=gen, dtype=torch.float64) - 0.5) * 0.2 for i, v in enumerate(vocab)}


def make_batch(gen, B, hot, vocab=(50, 7, 300), variable=True, power_law=False, ones=False):
    """keys [B, H] per input (-1 padding for a variable bag) and their fp32 weights: uniform in [-0.5, 1.5),
    NaN at padding positions (ignored, whatever the value), the first bag of each weighted multi-hot input
    summing to exactly 0; all 1.0 with ``ones``"""
    keys, wts = {}, {}
    for i, name in enumerate(INPUTS):
        H = hot[name]
        if power_law:
            from hugectr_b200.data.batch import power_law_keys
            k = power_law_keys(B * H, vocab[i], 1.2, gen).view(B, H)
        else:
            k = torch.randint(0, vocab[i], (B, H), generator=gen)
        if variable and H > 1:
            n = torch.randint(0, H + 1, (B,), generator=gen)
            n[0] = H
            k = torch.where(torch.arange(H).view(1, -1) < n.view(-1, 1), k, torch.full_like(k, -1))
        w = (torch.rand(B, H, generator=gen) * 2 - 0.5)
        if H >= 2:
            w[0, :] = 0
            w[0, 0], w[0, 1] = 0.75, -0.75
        if ones:
            w = torch.ones(B, H)
        w = torch.where(k >= 0, w, torch.full_like(w, float("nan")))
        keys[name], wts[name] = k, w
    return keys, wts


def flat(d, rows=None):
    """feature-major 1-D batch (the layout of set_keys / set_weights), optionally a row window"""
    return torch.cat([(v if rows is None else v[rows]).reshape(-1) for v in d.values()])


def _denom(name, k, w, combiner):
    valid = k >= 0
    if combiner != "mean":
        return torch.ones(k.shape[0], dtype=torch.float64)
    if name in WEIGHTED:
        sw = torch.where(valid, w.double(), torch.zeros((), dtype=torch.float64)).sum(1)
        return torch.where(sw == 0, torch.ones_like(sw), sw)
    return valid.sum(1).clamp(min=1).double()


def oracle_forward(tables, keys, wts, combiner):
    """fp64 pooled [B, 3 * ev] of the top "emb" from the semantics"""
    outs = []
    for i, name in enumerate(INPUTS):
        k, w = keys[name], wts[name]
        comb = combiner if name != "u1" else "sum"
        valid = k >= 0
        ww = torch.where(valid, w.double(), torch.zeros((), dtype=torch.float64)) if name in WEIGHTED \
            else valid.double()
        rows = tables[str(i)][k.clamp(min=0)]
        outs.append((ww.unsqueeze(-1) * rows).sum(1) / _denom(name, k, w, comb).unsqueeze(1))
    return torch.cat(outs, 1)


def oracle_grad(tables, keys, wts, combiner, grad):
    """fp64 summed gradient per table row of one step on the top gradient ``grad`` [B, 3 * ev]"""
    ev = tables["0"].shape[1]
    out = {}
    for i, name in enumerate(INPUTS):
        k, w = keys[name], wts[name]
        comb = combiner if name != "u1" else "sum"
        valid = k >= 0
        ww = torch.where(valid, w.double(), torch.zeros((), dtype=torch.float64)) if name in WEIGHTED \
            else valid.double()
        g = grad[:, i * ev:(i + 1) * ev].double() / _denom(name, k, w, comb).unsqueeze(1)
        contrib = (ww.unsqueeze(-1) * g.unsqueeze(1)).reshape(-1, ev)
        out[str(i)] = torch.zeros_like(tables[str(i)]).index_add_(0, k.clamp(min=0).reshape(-1),
                                                                   contrib * valid.reshape(-1, 1))
    return out


def oracle_sgd(tables, keys, wts, combiner, grad, lr):
    """fp64 tables after one SGD step"""
    d = oracle_grad(tables, keys, wts, combiner, grad)
    return {n: t - lr * d[n] for n, t in tables.items()}


def oracle_adagrad(tables, keys, wts, combiner, grad, lr, accu0, eps):
    """fp64 tables after one AdaGrad step from accumulators ``accu0``: s = accu0 + g^2, w -= lr g / (sqrt(s) + eps)"""
    d = oracle_grad(tables, keys, wts, combiner, grad)
    return {n: t - lr * d[n] / ((accu0 + d[n] * d[n]).sqrt() + eps) for n, t in tables.items()}


def dump_full(e, vocab, ev=16):
    """{table: fp64 [vocab, ev]} of the shards held by ``e`` (rows this rank does not hold are NaN)"""
    res = {}
    for i, v in enumerate(vocab):
        full = None
        for (k, w, c0, _, _) in e.dump_table_local(str(i)):
            if full is None:
                full = torch.full((v, ev), float("nan"), dtype=torch.float64)
            m = (k >= 0) & (k < v)
            full[k[m], c0:c0 + w.shape[1]] = w[m].double()
        res[str(i)] = full
    return res


def step(e, keys, wts, grad, lr=0.1, rows=None, weights=True):
    """one forward + backward of collection ``e`` on (a row window of) the batch; returns the output"""
    dev = e.device
    e.set_keys(flat(keys, rows).to(e.key_dtype).to(dev))
    if weights:
        e.set_weights(flat(wts, rows).to(dev))
    e.forward()
    out = e.top_data["emb"].float().cpu().clone()
    g = grad if rows is None else grad[rows]
    e.top_grad["emb"].copy_(g.to(dev))
    e.backward(torch.tensor([lr], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))
    return out


def check_tables(got, exp, atol):
    for n in exp:
        if got.get(n) is None:
            continue
        m = ~torch.isnan(got[n])
        err = (got[n][m] - exp[n][m]).abs().max().item() if bool(m.any()) else 0.0
        assert err < atol, f"table {n}: err {err}"


HOT = {"w0": 4, "u1": 1, "w2": 8}


# ----------------------------------------------------------------------------- fp64 oracle, one process
@pytest.mark.parametrize("combiner", ["sum", "mean"])
@pytest.mark.parametrize("variable", [False, True])
def test_cpu_matches_fp64_oracle(combiner, variable):
    gen = torch.Generator().manual_seed(11)
    B = 24
    tables = make_tables(gen)
    e = make_collection(CPU, Comm.single(CPU), B, HOT, combiner=combiner)
    load_tables(e, tables)
    exp_tabs = tables
    for it in range(2):
        keys, wts = make_batch(gen, B, HOT, variable=variable)
        if it == 0:
            # negative weights and a weight far from 1 on one bag
            wts["w2"][1] = torch.where(keys["w2"][1] >= 0, torch.linspace(-2, 3, HOT["w2"]), wts["w2"][1])
        grad = torch.randn(B, 48, generator=gen) * 0.1
        out = step(e, keys, wts, grad)
        exp = oracle_forward(exp_tabs, keys, wts, combiner)
        assert torch.isfinite(out).all()
        assert (out.double() - exp).abs().max().item() < 1e-5
        exp_tabs = oracle_sgd(exp_tabs, keys, wts, combiner, grad, 0.1)
        check_tables(dump_full(e, (50, 7, 300)), exp_tabs, 1e-6)


@pytest.mark.parametrize("combiner", ["sum", "mean"])
@pytest.mark.parametrize("plan", ["table", "dp"])
def test_adagrad_step_matches_fp64_oracle(combiner, plan, dev=CPU):
    """a stateful optimizer against the oracle directly (the GPU file runs this on the device)"""
    gen = torch.Generator().manual_seed(17)
    B = 32
    tables = make_tables(gen)
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-7)
    comm = Comm.single(dev)
    e = make_collection(dev, comm, B, HOT, plan=plan, combiner=combiner, opt=opt)
    load_tables(e, tables)
    keys, wts = make_batch(gen, B, HOT)
    grad = torch.randn(B, 48, generator=gen) * 0.1
    step(e, keys, wts, grad, lr=0.1)
    check_tables(dump_full(e, (50, 7, 300)), oracle_adagrad(tables, keys, wts, combiner, grad, 0.1, 0.1, 1e-7), 2e-6)


def test_zero_sum_mean_divides_by_one():
    gen = torch.Generator().manual_seed(2)
    tables = make_tables(gen)
    e = make_collection(CPU, Comm.single(CPU), 4, HOT, combiner="mean")
    load_tables(e, tables)
    keys, wts = make_batch(gen, 4, HOT, variable=False)
    e.set_keys(flat(keys).int()); e.set_weights(flat(wts)); e.forward()
    out = e.top_data["emb"].double()
    k = keys["w0"][0]
    exp = 0.75 * tables["0"][k[0]] - 0.75 * tables["0"][k[1]]        # sum_w == 0: divided by 1
    assert (out[0, :16] - exp).abs().max().item() < 1e-6


# ----------------------------------------------------------------------------- all ones == unweighted, bit for bit
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_all_ones_equal_unweighted_cpu(combiner):
    gen = torch.Generator().manual_seed(4)
    B = 16
    tables = make_tables(gen)
    opt = CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1, epsilon=1e-7)
    ew = make_collection(CPU, Comm.single(CPU), B, HOT, combiner=combiner, opt=opt)
    eu = make_collection(CPU, Comm.single(CPU), B, HOT, combiner=combiner, opt=opt, weighted=())
    load_tables(ew, tables); load_tables(eu, tables)
    for _ in range(2):
        keys, wts = make_batch(gen, B, HOT, ones=True)
        grad = torch.randn(B, 48, generator=gen) * 0.1
        ow = step(ew, keys, wts, grad)
        eu.set_keys(flat(keys).int()); eu.forward()
        ou = eu.top_data["emb"].clone()
        eu.top_grad["emb"].copy_(grad)
        eu.backward(torch.tensor([0.1]), torch.tensor([1], dtype=torch.int32))
        assert torch.equal(ow, ou)
    for gw, gu in zip(ew.groups, eu.groups):
        assert torch.equal(gw.table, gu.table) and torch.equal(gw.s0, gu.s0)


# ----------------------------------------------------------------------------- emulated ranks == one process
@pytest.mark.parametrize("plan", ["table", "row", "column", "dp"])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_emulated_ranks_equal_one_process(plan, combiner):
    from hugectr_b200.parallel.emu import run_ranks
    world, b = 2, 8
    gen = torch.Generator().manual_seed(21)
    tables = make_tables(gen)
    batches = [make_batch(gen, b * world, HOT) + (torch.randn(b * world, 48, generator=gen) * 0.1,) for _ in range(2)]
    one = make_collection(CPU, Comm.single(CPU), b * world, HOT, combiner=combiner)
    load_tables(one, tables)
    ref_out = [step(one, k, w, g) for (k, w, g) in batches]
    ref_tab = dump_full(one, (50, 7, 300))

    def rank_fn(comm):
        e = make_collection(CPU, comm, b, HOT, plan=plan, combiner=combiner, fused=False)
        load_tables(e, tables)
        rows = slice(comm.rank * b, (comm.rank + 1) * b)
        for (k, w, g), ro in zip(batches, ref_out):
            out = step(e, k, w, g, rows=rows)
            assert (out - ro[rows]).abs().max().item() < 1e-6
        comm.barrier()
        check_tables(dump_full(e, (50, 7, 300)), ref_tab, 1e-6)
        return True
    assert all(run_ranks(world, rank_fn, device=CPU))


# ----------------------------------------------------------------------------- rejections
def test_rejections():
    t = EmbeddingTableConfig("t", 10, 4)
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(t, "w0", "top", "concat")
    with pytest.raises(ValueError, match="w0"):
        EmbeddingCollection(cfg, 4, {"w0": 2}, CPU, torch.float32, Comm.single(CPU),
                            CreateOptimizer(Optimizer_t.SGD), weighted={"w0"})
    from hugectr_b200.parallel.emu import run_ranks
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(t, "w0", "top", "sum")
    cfg.shard([[1], [1]], [("mp", ["t"])], {CompressionStrategy.Unique: ["t"]})

    def mk(comm):
        with pytest.raises(ValueError, match="table t"):
            EmbeddingCollection(cfg, 4, {"w0": 2}, CPU, torch.float32, comm, CreateOptimizer(Optimizer_t.SGD),
                                weighted={"w0"}, fused=False)
        return True
    assert all(run_ranks(2, mk, device=CPU))


def _model(tmp_path, reader_type=None, legacy=False, weighted=True, source=("synthetic",), device=CPU):
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]],
                                  use_cuda_graph=device.type == "cuda")
    rp = hugectr.DataReaderParams(reader_type or hugectr.DataReaderType_t.Parquet, source=list(source),
                                  eval_source=source[0], check_type=hugectr.Check_t.Non,
                                  slot_size_array=[100, 20])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad), comm=Comm.single(device))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[
                            hugectr.DataReaderSparseParam("a", 3, False, 1, weighted=weighted),
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


def test_model_rejections(tmp_path):
    for t in (hugectr.DataReaderType_t.Norm, hugectr.DataReaderType_t.Raw, hugectr.DataReaderType_t.RawAsync):
        with pytest.raises(ValueError, match="weighted input a"):
            _model(tmp_path, reader_type=t).compile()
    with pytest.raises(ValueError, match="weighted input a"):
        _model(tmp_path, legacy=True).compile()


# ----------------------------------------------------------------------------- graph JSON
def test_graph_json_round_trip(tmp_path):
    from hugectr_b200.graph_json import model_to_json
    m = _model(tmp_path)
    j = model_to_json(m)
    sp = {s["top"]: s for s in j["layers"][0]["sparse"]}
    assert sp["a"]["weighted"] is True and "weighted" not in sp["b"]
    path = tmp_path / "g.json"
    path.write_text(json.dumps(j))
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["synthetic"], eval_source="synthetic",
                                  check_type=hugectr.Check_t.Non, slot_size_array=[100, 20])
    m2 = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m2.construct_from_json(str(path))
    prm = {p.top_name: p for p in m2.input.data_reader_sparse_param_array}
    assert prm["a"].weighted and not prm["b"].weighted
    assert "weighted" not in hugectr.DataReaderSparseParam("x", 2, True, 1).to_json()


# ----------------------------------------------------------------------------- readers and a weighted model
def test_synthetic_reader_streams_unchanged():
    from hugectr_b200.data.readers import SparseLayout, SyntheticReader
    from hugectr_b200.solver import DataReaderSparseParam as P
    mk = lambda w: SyntheticReader(16, 0, 1, 1, 3, SparseLayout([P("a", 3, False, 1, weighted=w), P("b", 1, True, 1)]),
                                   [100, 20], seed=5, pool=2)
    r0, r1 = mk(False), mk(True)
    for h0, h1 in zip(r0.pool, r1.pool):
        assert torch.equal(h0.keys, h1.keys) and torch.equal(h0.label, h1.label) and torch.equal(h0.dense, h1.dense)
        assert h0.weights is None and h1.weights.shape == h1.keys.shape
        assert float(h1.weights[:48].min()) >= 0.5 and float(h1.weights[:48].max()) < 1.5
        assert bool((h1.weights[48:] == 1).all())
        assert h1.h2d_bytes() == h0.h2d_bytes() + h1.weights.numel() * 4


def test_weighted_synthetic_model_trains(tmp_path):
    m = _model(tmp_path)
    m.compile()
    m.fit(max_iter=8, display=100, eval_interval=100)
    e = m.ebcs_train[0]
    assert e.has_weights and float(e.weight_slab.min()) >= 0.5
    assert np.isfinite(m.get_current_loss())


# ----------------------------------------------------------------------------- Parquet weight columns
def write_weighted_parquet(d, sizes, seed, row_group_size=7, mismatch=False, weight_index=True):
    """files of label, 2 dense, a (list<int64>, 0..5 keys: empty and over-long bags), its list<float> weights,
    b (int64, unweighted), c (int64 one-hot) and its float weights; returns (file list, rows)"""
    import pyarrow as pa
    import pyarrow.parquet as pq
    rng = np.random.default_rng(seed)
    files, rows = [], []
    for f, n in enumerate(sizes):
        cnt = rng.integers(0, 6, n)
        a = [rng.integers(0, 100, c).tolist() for c in cnt]
        aw = [rng.uniform(-1, 2, c).astype("float32").tolist() for c in cnt]
        if mismatch:
            aw[n // 2] = aw[n // 2] + [1.0]
        bb, cc = rng.integers(0, 20, n), rng.integers(0, 100, n)
        cw = rng.uniform(-1, 2, n).astype("float32")
        cols = [pa.array(rng.integers(0, 2, n).astype("float32")), pa.array(rng.random(n, dtype=np.float32)),
                pa.array(rng.random(n, dtype=np.float32)), pa.array(a, type=pa.list_(pa.int64())),
                pa.array(aw, type=pa.list_(pa.float32())), pa.array(bb), pa.array(cc), pa.array(cw)]
        path = os.path.join(d, f"p{f}.parquet")
        pq.write_table(pa.Table.from_arrays(cols, names=["l", "d0", "d1", "a", "a_w", "b", "c", "c_w"]), path,
                       row_group_size=row_group_size)
        files.append(path)
        rows += [(a[i], aw[i], int(bb[i]), int(cc[i]), float(cw[i])) for i in range(n)]
    cats = [{"index": 3, "weight_index": 4}, {"index": 5}, {"index": 6, "weight_index": 7}]
    if not weight_index:
        del cats[2]["weight_index"]
    json.dump({"file_stats": [], "labels": [{"index": 0}], "conts": [{"index": 1}, {"index": 2}], "cats": cats},
              open(os.path.join(d, "_metadata.json"), "w"))
    fl = os.path.join(d, "fl.txt")
    open(fl, "w").write(f"{len(files)}\n" + "\n".join(files) + "\n")
    return fl, rows


def _reader(fl, b, rank, world, weighted=(True, False, True)):
    from types import SimpleNamespace as NS
    from hugectr_b200.data.parquet_reader import ParquetReader
    layout = NS(blocks=[("a", 1, 3, False), ("b", 1, 1, True), ("c", 1, 1, True)], total_slots=3, weighted=list(weighted))
    model = NS(reader_params=NS(source=[fl], eval_source=fl, slot_size_array=[], num_workers=2), b_train=b, b_eval=b,
               comm=NS(rank=rank), world=world, input=NS(label_dim=1, dense_dim=2), layout=layout,
               key_dtype=torch.int32, solver=NS(repeat_dataset=False), sparse_embeddings=[], device=CPU)
    return ParquetReader(model, True)


@pytest.mark.parametrize("world", [1, 2])
def test_parquet_reader_delivers_the_weights(tmp_path, world):
    """one-hot and multi-hot weighted slots, batches across row-group and file boundaries, the incomplete last batch"""
    b, H = 5, 3
    fl, rows = write_weighted_parquet(str(tmp_path), [23, 16], seed=world)
    gb = b * world
    nbatches = 0
    for rank in range(world):
        r = _reader(fl, b, rank, world)
        r.start()
        bi = 0
        while True:
            hb = r.read_a_batch()
            if hb is None:
                break
            k, w = hb.keys.numpy(), hb.weights.numpy()
            assert hb.weights.dtype == torch.float32 and w.shape == k.shape
            ka, kb, kc = k[:b * H].reshape(b, H), k[b * H:b * H + b], k[b * H + b:]
            wa, wb, wc = w[:b * H].reshape(b, H), w[b * H:b * H + b], w[b * H + b:]
            for i in range(b):
                g = bi * gb + rank * b + i
                if g >= len(rows):                       # behind the incomplete last batch: padding
                    assert (ka[i] == -1).all() and (wa[i] == 0).all() and kc[i] == -1 and wc[i] == 0
                    continue
                a, aw, bb, cc, cw = rows[g]
                m = min(len(a), H)
                assert ka[i, :m].tolist() == a[:m] and (ka[i, m:] == -1).all()
                assert wa[i, :m].tolist() == aw[:m] and (wa[i, m:] == 0).all()
                assert kb[i] == bb and wb[i] == 1.0
                assert kc[i] == cc and wc[i] == np.float32(cw)
            bi += 1
        r.stop()
        nbatches = bi
    assert nbatches == (len(rows) + gb - 1) // gb and len(rows) % gb


def test_parquet_reader_rejects_bad_weight_columns(tmp_path):
    d1, d2 = tmp_path / "nowi", tmp_path / "mismatch"
    d1.mkdir(); d2.mkdir()
    fl, _ = write_weighted_parquet(str(d1), [10], seed=0, weight_index=False)
    with pytest.raises(ValueError, match="weighted input c: slot 0 .* has no weight_index"):
        _reader(fl, 4, 0, 1)
    fl, _ = write_weighted_parquet(str(d2), [10], seed=0, mismatch=True, row_group_size=4)
    r = _reader(fl, 4, 0, 1)
    r.start()
    with pytest.raises(ValueError, match=r"p0.parquet row group 1: weight column a_w .* key column a"):
        while r.read_a_batch() is not None:
            pass
    r.stop()


def test_weighted_parquet_model_trains(tmp_path):
    fl, rows = write_weighted_parquet(str(tmp_path), [40, 33], seed=3, row_group_size=16)
    m = _model(tmp_path, source=(fl,))
    m.compile()
    m.fit(max_iter=6, display=100, eval_interval=100)
    e = m.ebcs_train[0]
    assert e.has_weights and not bool((e.weight_slab == 1).all())
    assert np.isfinite(m.get_current_loss())
