"""Delta export of embedding-collection tables (EmbeddingTableConfig(track_updates=True),
Model.embedding_dump_delta, InferenceModel.update_embedding) on the CPU path: validation, graph JSON, the exact
delta of a model against a host oracle of the batches, the serving round trip, and emulated ranks whose delta
folders are byte-identical to the one-rank delta."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                               EmbeddingTableConfig)
from hugectr_b200.embedding.hashtable import AdmitSketch
from hugectr_b200.enums import CompressionStrategy, Optimizer_t
from hugectr_b200.inference import InferenceModel, InferenceParams
from hugectr_b200.io.checkpoint import embedding_dump_delta, read_delta_info, read_ebc_folder, save_dense
from hugectr_b200.model import Model
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

CPU = torch.device("cpu")
B, EV = 32, 8
# model of the exact-delta tests: (input, hotness, table, combiner); table "c" is dynamic, "w" weighted
INPUTS = [("a", 2, "ta", "sum"), ("b", 3, "tb", "mean"), ("c", 2, "tc", "sum"), ("w", 2, "tw", "sum")]
VOCAB = {"ta": 500, "tb": 300, "tw": 400}
DYN_BASE = 10 ** 12
DYN_CAP = 4096


def tables(track=True):
    return [EmbeddingTableConfig("ta", VOCAB["ta"], EV, track_updates=track),
            EmbeddingTableConfig("tb", VOCAB["tb"], EV, weight_dtype="bf16", track_updates=track,
                                 opt_params=CreateOptimizer(Optimizer_t.RowWiseAdaGrad, initial_accu_value=0.1)),
            EmbeddingTableConfig("tc", -1, EV, init_capacity=DYN_CAP, admit_threshold=2, track_updates=track),
            EmbeddingTableConfig("tw", VOCAB["tw"], EV, track_updates=track)]


def build_model(device=CPU, track=True, graph=False, seed=5, weighted=True):
    """the model of INPUTS; ``weighted``: input "w" carries per-key weights (serving sessions take keys only)"""
    solver = hugectr.CreateSolver(batchsize=B, batchsize_eval=B, lr=0.05, vvgpu=[[0]], repeat_dataset=True,
                                  i64_input_key=True, use_cuda_graph=graph, seed=seed)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["synthetic"],
                                  eval_source="synthetic", check_type=hugectr.Check_t.Non,
                                  slot_size_array=[VOCAB["ta"], VOCAB["tb"], 300, VOCAB["tw"]])
    m = Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad, initial_accu_value=0.1),
              comm=Comm.single(device))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam(n, h, False, 1, weighted=weighted and n == "w")
                                                        for n, h, _, _ in INPUTS]))
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(tables(track), [n for n, _, _, _ in INPUTS], "emb", [c for _, _, _, c in INPUTS])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["cat"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["cat"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    return m


def batches(n, seed=3, distinct=False):
    """host batches: power-law keys with padding (-1), the dynamic table's keys far above 2^32; ``distinct``: every
    key occurs at most once per input and batch (uniform keys instead)"""
    from hugectr_b200.data.batch import HostBatch
    rng = np.random.default_rng(seed)
    res = []
    for _ in range(n):
        keys, per = [], {}
        for name, h, t, _ in INPUTS:
            hi = VOCAB.get(t, 300)
            if distinct:
                k = rng.permutation(hi)[:B * h].reshape(B, h).astype(np.int64)
            else:
                k = np.minimum((rng.pareto(1.1, (B, h)) * 15).astype(np.int64), hi - 1)
            k[rng.random((B, h)) < 0.15] = -1
            if t == "tc":
                k = np.where(k >= 0, k + DYN_BASE, -1)
            per[name] = k
            keys.append(k.reshape(-1))
        w = [np.ones(B * h, dtype=np.float32) if n != "w" else rng.uniform(0.25, 2.0, B * h).astype(np.float32)
             for n, h, _, _ in INPUTS]
        hb = HostBatch(torch.from_numpy(rng.integers(0, 2, (B, 1)).astype(np.float32)),
                       torch.from_numpy(rng.standard_normal((B, 2)).astype(np.float32)),
                       torch.from_numpy(np.concatenate(keys)), None, B,
                       weights=torch.from_numpy(np.concatenate(w)))
        res.append((hb, per))
    return res


def rows_given(bs, lo, hi):
    """{table: set of keys} that steps lo+1..hi (1-based) gave rows, from the batches alone: every valid key of a
    static table; for the admitting dynamic table the keys present or admitted that step, replayed with the CPU
    sketch (hashtable.py::AdmitSketch) from step 1"""
    sk = AdmitSketch(DYN_CAP, 2, 0, torch.zeros(1, dtype=torch.int64), CPU)
    present, res = set(), {t: set() for _, _, t, _ in INPUTS}
    for step, (_, per) in enumerate(bs[:hi], 1):
        got = {}
        for name, _, t, _ in INPUTS:
            k = [int(x) for x in per[name].reshape(-1) if x >= 0]
            if t != "tc":
                got[t] = set(k)
                continue
            miss = [x for x in k if x not in present]
            sk.count(miss)
            adm = {x for x, ok in zip(miss, sk.admits(miss)) if ok}
            present |= adm
            got[t] = {x for x in k if x in present}
        if step > lo:
            for t, s in got.items():
                res[t] |= s
    return res


def by_key(folder):
    """{table name: {key: fp32 row}} of an embedding_collection_0 folder"""
    names = [t for _, _, t, _ in INPUTS]
    out = {}
    for tid, (k, w, _) in read_ebc_folder(f"{folder}/embedding_collection_0").items():
        out[names[tid]] = {int(x): w[i] for i, x in enumerate(k.tolist())}
    return out


def check_exact_delta(device, tmp, graph):
    """train to A, full dump + clocks, train to B, delta since A: the oracle's keys, every changed row, the bytes
    of the full dump at B"""
    m = build_model(device, graph=graph)
    bs = batches(9)
    A, Bstep = 4, 9
    for hb, _ in bs[:A]:
        m.train_on_host_batch(hb)
    since = m.embedding_clocks()
    assert since == {0: A}
    m.embedding_dump(f"{tmp}/full_a")
    for hb, _ in bs[A:Bstep]:
        m.train_on_host_batch(hb)
    until = m.embedding_dump_delta(f"{tmp}/delta", since)
    assert until == {0: Bstep} == m.embedding_clocks()
    m.embedding_dump(f"{tmp}/full_b")
    info = read_delta_info(f"{tmp}/delta")
    assert info == {0: {"since": A, "until": Bstep, "tables": ["ta", "tb", "tc", "tw"], "data_parallel": []}}
    want = rows_given(bs, A, Bstep)
    d, fa, fb = by_key(f"{tmp}/delta"), by_key(f"{tmp}/full_a"), by_key(f"{tmp}/full_b")
    for _, _, t, _ in INPUTS:
        assert set(d[t]) == want[t], t
        assert list(d[t]) == sorted(d[t]), t
        changed = {k for k, v in fb[t].items() if k not in fa[t] or not torch.equal(v, fa[t][k])}
        assert changed and changed <= set(d[t]), t
        for k, v in d[t].items():
            assert torch.equal(v, fb[t][k]), (t, k)
    # the delta folder loads through embedding_load as any checkpoint
    m2 = build_model(device, seed=77)
    m2.embedding_load(f"{tmp}/full_a")
    m2.embedding_load(f"{tmp}/delta")
    m2.embedding_dump(f"{tmp}/full_m2")
    assert by_key(f"{tmp}/full_m2").keys() == fb.keys()
    for t, rows in by_key(f"{tmp}/full_m2").items():
        assert rows.keys() == fb[t].keys() and all(torch.equal(v, fb[t][k]) for k, v in rows.items())
    return m


def predict_batches(n=3, seed=11):
    rng = np.random.default_rng(seed)
    res = []
    for _ in range(n):
        keys = []
        for _, h, t, _ in INPUTS:
            k = rng.integers(0, VOCAB.get(t, 300), B * h)
            keys.append(k + DYN_BASE if t == "tc" else k)
        res.append((rng.standard_normal((B, 2)).astype(np.float32), np.concatenate(keys).astype(np.int64)))
    return res


def check_serving_round_trip(device, tmp, graph):
    """session 1: full dump at A + deltas A->B and B->C (C through fit); session 2: full dump at C.  Same tables,
    same predictions, with fp8_quant off and on.  A gap raises, an overlap does not."""
    m = build_model(device, graph=graph, weighted=False)
    bs = batches(6, seed=4)
    for hb, _ in bs[:3]:
        m.train_on_host_batch(hb)
    ca = m.embedding_clocks()
    m.embedding_dump(f"{tmp}/full_a")
    for hb, _ in bs[3:]:
        m.train_on_host_batch(hb)
    cb = m.embedding_dump_delta(f"{tmp}/d_ab", ca)
    m.fit(max_iter=4, display=0, eval_interval=0, snapshot=0, delta_interval=4, delta_prefix=f"{tmp}/d_fit_")
    info = read_delta_info(f"{tmp}/d_fit_4")
    assert info[0]["since"] == cb[0] and info[0]["until"] == cb[0] + 4
    cc = m.embedding_clocks()
    m.embedding_dump(f"{tmp}/full_c")
    save_dense(m, f"{tmp}/dense", 0)
    m.graph_to_json(f"{tmp}/graph.json")
    for hb, _ in batches(2, seed=5):
        m.train_on_host_batch(hb)
    m.embedding_dump_delta(f"{tmp}/d_cd", cc)
    dev = str(device)
    for fp8 in (False, True):
        p = dict(model_name="delta", max_batchsize=B, dense_model_file=f"{tmp}/dense_dense_0.model",
                 i64_input_key=True, fp8_quant=fp8)
        s1 = InferenceModel(f"{tmp}/graph.json", InferenceParams(**p, embedding_collection_path=f"{tmp}/full_a"), dev)
        s1.update_embedding(f"{tmp}/d_ab")
        with pytest.raises(ValueError, match=r"collection 0 .*clock 10.*clock 6"):
            s1.update_embedding(f"{tmp}/d_cd")           # C -> D onto a session at B < C: a gap
        s1.update_embedding(f"{tmp}/d_ab")               # an overlap is fine
        s1.update_embedding(f"{tmp}/d_fit_4")
        assert s1.delta_clocks == {0: cc[0]}
        with pytest.raises(ValueError, match=r"collection 0 ends at clock 6.*clock 10: .*roll rows back"):
            s1.update_embedding(f"{tmp}/d_ab")           # A -> B onto a session at C > B: older rows
        assert s1.delta_clocks == {0: cc[0]}
        s2 = InferenceModel(f"{tmp}/graph.json", InferenceParams(**p, embedding_collection_path=f"{tmp}/full_c"), dev)
        s1.model.embedding_dump(f"{tmp}/s1_{fp8}")
        s2.model.embedding_dump(f"{tmp}/s2_{fp8}")
        t1, t2 = by_key(f"{tmp}/s1_{fp8}"), by_key(f"{tmp}/s2_{fp8}")
        assert t1.keys() == t2.keys()
        for t in t1:
            assert t1[t].keys() == t2[t].keys(), t
            assert all(torch.equal(v, t2[t][k]) for k, v in t1[t].items()), t
        for dense, keys in predict_batches():
            assert np.array_equal(s1.predict(dense, keys), s2.predict(dense, keys))


# ----------------------------------------------------------------------------- validation and graph JSON
@pytest.mark.parametrize("v", [1, "yes", None, 1.0])
def test_track_updates_takes_a_bool_only(v):
    with pytest.raises(ValueError, match="table tt: track_updates must be a bool"):
        EmbeddingTableConfig("tt", 10, 8, track_updates=v)


def test_track_updates_rejects_an_evicting_table():
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(EmbeddingTableConfig("ev", -1, 8, max_capacity=64, evict_strategy="lru", track_updates=True),
                         "k", "emb", "sum")
    with pytest.raises(ValueError, match="table ev: track_updates does not support an evicting table"):
        EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, Comm.single(CPU),
                            CreateOptimizer(Optimizer_t.SGD), key_dtype=torch.int64)


def test_graph_json_round_trips_track_updates(tmp_path):
    m = build_model()
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    tj = [l for l in json.load(open(p))["layers"] if l["type"] == "EmbeddingCollection"][0]["tables"]
    assert all(t["track_updates"] is True for t in tj)
    m2 = Model(hugectr.CreateSolver(batchsize=B, batchsize_eval=B, vvgpu=[[0]], i64_input_key=True,
                                    use_cuda_graph=False), m.reader_params, hugectr.CreateOptimizer(Optimizer_t.SGD),
               comm=Comm.single(CPU))
    m2.construct_from_json(p)
    assert all(t.track_updates for t in m2.ebc_configs[0].tables())
    p2 = str(tmp_path / "g2.json")
    m2.compile()
    m2.graph_to_json(p2)
    assert open(p, "rb").read() == open(p2, "rb").read()
    build_model(track=False).graph_to_json(str(tmp_path / "g3.json"))
    assert b"track_updates" not in open(str(tmp_path / "g3.json"), "rb").read()


def test_tracking_off_allocates_no_stamps_and_keeps_the_clock():
    m = build_model(track=False)
    e = m.ebcs_train[0]
    assert all(g.stamp is None for g in e.groups)
    assert e.ticks_clock                                   # (the admitting table ticks it)
    e2 = build_model(track=True).ebcs_train[0]
    stamps = sum(g.stamp.numel() * 4 for g in e2.groups if g.stamp is not None)
    assert stamps == 4 * sum(g.rows for g in e2.groups) and e2.memory_bytes() == e.memory_bytes() + stamps
    with pytest.raises(ValueError, match="table ta: it does not track updates"):
        e.delta_table_local("ta", 0)


def test_static_tracked_collection_ticks_its_clock():
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(EmbeddingTableConfig("s", 40, 8, track_updates=True), "k", "emb", "sum")
    e = EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, Comm.single(CPU),
                            CreateOptimizer(Optimizer_t.SGD), key_dtype=torch.int64)
    assert e.ticks_clock and e.groups[0].stamp is not None
    train_step(e, [3, 7, -1, 3])
    train_step(e, [9, -1, -1, 39])
    assert int(e.evict_clock) == 2
    st = e.groups[0].stamp
    assert {i: int(st[i]) for i in range(40) if st[i]} == {3: 1, 7: 1, 9: 2, 39: 2}
    e.load_table_rows("s", torch.tensor([5, 9]), torch.ones(2, 8))
    assert int(st[5]) == int(st[9]) == 3                    # clock + 1: a delta since the clock holds them
    ((k, w, c0, sts, kind),) = e.delta_table_local("s", 1)
    assert k.tolist() == [5, 9, 39] and torch.equal(w[:2], torch.ones(2, 8)) and sts == [] and kind == "mp"


def test_growth_relays_the_stamps():
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig("d", -1, 8, init_capacity=4, track_updates=True),
                          EmbeddingTableConfig("s", 10, 8, track_updates=True)], ["k", "j"], "emb", ["sum", "sum"])
    e = EmbeddingCollection(cfg, 4, {"k": 1, "j": 1}, CPU, torch.float32, Comm.single(CPU),
                            CreateOptimizer(Optimizer_t.SGD), key_dtype=torch.int64)
    train_step(e, [100, 101, 102, 103, 1, 2, -1, -1])
    train_step(e, [104, 105, -1, -1, 3, -1, -1, -1])       # the shard is full: 104, 105 get no row
    assert e.grow_dynamic()
    grp = e.groups[0]
    assert grp.stamp.numel() == grp.rows
    train_step(e, [104, -1, -1, -1, -1, -1, -1, -1])
    ((dk, *_),), ((sk, *_),) = e.delta_table_local("d", 0), e.delta_table_local("s", 1)
    assert dk.tolist() == [100, 101, 102, 103, 104] and sk.tolist() == [3]
    assert e.delta_table_local("d", 2)[0][0].tolist() == [104]


def train_step(e, keys, grads=None, lr=0.05):
    dev = e.device
    e.set_keys(torch.as_tensor(keys, dtype=torch.int64).to(dev))
    e.forward(True)
    g = e.top_grad["emb"]
    g.copy_(((0.5 * e.top_data["emb"] + 0.01) if grads is None else grads).to(g.dtype))
    e.backward(torch.tensor([lr], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))


# ----------------------------------------------------------------------------- the model on the CPU path
def test_exact_delta_cpu(tmp_path):
    check_exact_delta(CPU, str(tmp_path), graph=False)


def test_serving_round_trip_cpu(tmp_path):
    check_serving_round_trip(CPU, str(tmp_path), graph=False)


def test_update_embedding_rejects_a_table_the_session_lacks(tmp_path):
    tmp = str(tmp_path)
    m = build_model(weighted=False)
    m.embedding_dump(f"{tmp}/full")
    m.graph_to_json(f"{tmp}/graph.json")
    save_dense(m, f"{tmp}/dense", 0)
    m.embedding_dump_delta(f"{tmp}/d", None)
    s = InferenceModel(f"{tmp}/graph.json", InferenceParams("x", B, dense_model_file=f"{tmp}/dense_dense_0.model",
                                                            i64_input_key=True, embedding_collection_path=f"{tmp}/full"),
                       "cpu")
    info = json.load(open(f"{tmp}/d/delta.json"))
    info["collections"]["0"]["tables"].append("nope")
    json.dump(info, open(f"{tmp}/d/delta.json", "w"))
    with pytest.raises(ValueError, match="table nope of embedding collection 0 is not in this session"):
        s.update_embedding(f"{tmp}/d")


# ----------------------------------------------------------------------------- emulated ranks
EMU_ROWS = {"t0": 120, "t1": 90, "t3": 20}
EMU_HOT = {"k0": 2, "k1": 3, "k2": 2, "k3": 1}
EMU_DYN = [7 * i for i in range(60)]   # keys of t2 (plus DYN_BASE when it is dynamic)


def emu_cfg(world, plan, unique, dynamic):
    ts = [EmbeddingTableConfig("t0", EMU_ROWS["t0"], EV, track_updates=True),
          EmbeddingTableConfig("t1", EMU_ROWS["t1"], EV, track_updates=True),
          EmbeddingTableConfig("t2", -1 if dynamic else 7 * len(EMU_DYN), EV, init_capacity=256,
                               track_updates=True),
          EmbeddingTableConfig("t3", EMU_ROWS["t3"], EV, track_updates=True)]
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(ts, list(EMU_HOT), "emb", ["sum"] * 4)
    sm = [[0] * 4 for _ in range(world)]
    if plan == "table":
        for i in range(3):
            sm[i % world][i] = 1
        mp = ["t0", "t1", "t2"]
    elif plan == "row":
        for g in range(world):
            sm[g][0] = sm[g][1] = sm[g][2] = 1
        mp = ["t0", "t1", "t2"]
    else:                       # column-wise t0 over every rank, t1 row-wise, t2 on rank 0
        for g in range(world):
            sm[g][0] = sm[g][1] = 1
        sm[0][2] = 1
        mp = [("t0", world), "t1", "t2"]
    for g in range(world):
        sm[g][3] = 1
    cfg.shard(sm, [("mp", mp), ("dp", ["t3"])],
              compression_strategy={CompressionStrategy.Unique: ["t1"]} if unique else None)
    return cfg


def emu_run(comm, plan, fused, unique, folder, dynamic=True):
    """load every table with fixed values (initial values depend on the plan), train on exact dyadic gradients
    (their sums do not depend on the order), write the delta since step 2 after step 5"""
    world, rank = comm.world_size, comm.rank
    b = 16 // world
    e = EmbeddingCollection(emu_cfg(world, plan, unique, dynamic), b, EMU_HOT, CPU, torch.float32, comm,
                            CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.5), key_dtype=torch.int64,
                            seed=1, fused=fused)
    gen = torch.Generator().manual_seed(4)
    for n, rows in EMU_ROWS.items():
        e.load_table_rows(n, torch.arange(rows), torch.randint(-64, 64, (rows, EV), generator=gen).float() / 256)
    base = DYN_BASE if dynamic else 0
    e.load_table_rows("t2", base + torch.tensor(EMU_DYN), torch.randint(-64, 64, (len(EMU_DYN), EV), generator=gen) / 256.)
    shim = SimpleNamespace(comm=comm, world=world, ebcs_train=[e], key_dtype=torch.int64)
    shim.embedding_clocks = lambda: Model.embedding_clocks(shim)
    since = None
    for step in range(5):
        blocks = []
        for n, h in EMU_HOT.items():
            hi = {"k0": 40, "k1": EMU_ROWS["t1"], "k2": 25, "k3": EMU_ROWS["t3"]}[n]
            k = torch.randint(0, hi, (16, h), generator=gen)
            k[torch.rand(16, h, generator=gen) < 0.2] = -1
            if n == "k2":
                k = torch.where(k >= 0, base + 7 * k, k)
            blocks.append(k[rank * b:(rank + 1) * b].reshape(-1))
        grads = torch.randint(-8, 8, (16, 4 * EV), generator=gen).float() / 64
        train_step(e, torch.cat(blocks), grads[rank * b:(rank + 1) * b], lr=0.125)
        if step == 1:
            since = shim.embedding_clocks()
    if plan == "column":
        # the column slices of a key are stamped in the same steps
        ks = [p[0] for p in e.delta_table_local("t0", since[0])]
        allk = comm.all_gather_object(ks)
        flat = [k for r in allk for k in r]
        assert all(torch.equal(k, flat[0]) for k in flat), "column slices of t0 disagree"
    return embedding_dump_delta(shim, folder, since)


def folder_bytes(folder):
    out = {}
    for root, _, files in os.walk(folder):
        for f in files:
            out[os.path.relpath(os.path.join(root, f), folder)] = open(os.path.join(root, f), "rb").read()
    return out


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("plan,fused,unique", [("table", False, False), ("row", False, False),
                                               ("column", False, False), ("table", True, False),
                                               ("row", True, False), ("column", True, False),
                                               ("row", False, True)])
def test_emulated_ranks_write_the_one_rank_delta(tmp_path, world, plan, fused, unique):
    from hugectr_b200.parallel.emu import run_ranks
    one = str(tmp_path / "one")
    many = str(tmp_path / "many")
    # (the peer-memory flow runs on the CPU for static tables: table t2 is then static over the same keys)
    run_ranks(1, lambda c: emu_run(c, plan, False, False, one, dynamic=not fused), device=CPU, p2p=False)
    run_ranks(world, lambda c: emu_run(c, plan, fused, unique, many, dynamic=not fused), device=CPU,
              p2p="force" if fused else False)
    a, b = folder_bytes(one), folder_bytes(many)
    assert a == b
    info = json.loads(a["delta.json"])["collections"]["0"]
    assert info["data_parallel"] == ["t3"] and info["since"] == 2 and info["until"] == 5
    dp = read_ebc_folder(f"{one}/embedding_collection_0")[3][0]
    assert dp.tolist() == list(range(EMU_ROWS["t3"]))       # a data-parallel table is written whole
    d = read_ebc_folder(f"{one}/embedding_collection_0")
    assert 0 < d[0][0].numel() < 40 and 0 < d[2][0].numel() <= len(EMU_DYN)
