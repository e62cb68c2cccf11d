"""Admission of new keys to dynamic tables (EmbeddingTableConfig(admit_threshold=N, admit_decay_steps=P)) on the
CPU path: validation, graph JSON, the rules by hand, the collection against the same table fed a stream filtered
by a plain-Python model of the rules, threshold 1 against no option, row-sharded emulated ranks, checkpoints,
weighted inputs and Model.fit."""
import json

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                               EmbeddingTableConfig)
from hugectr_b200.embedding.hashtable import AdmitSketch, sketch_slots
from hugectr_b200.enums import Optimizer_t
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

from test_embedding_evict_cpu import power_law_batches

CPU = torch.device("cpu")
KINDS = ["growing", "lru", "lfu"]


def table(kind, name="t", cap=256, **kw):
    ev = dict(max_capacity=cap, evict_strategy=kind) if kind in ("lru", "lfu") else dict(init_capacity=cap)
    return EmbeddingTableConfig(name, -1, 8, **ev, **kw)


def collection(comm, kind, b, H, cap=256, opt=None, seed=7, wdtype="fp32", lookups=2, weighted=(),
               key_dtype=torch.int64, **kw):
    """one dynamic table row-sharded over every rank, ``lookups`` sum lookups of it"""
    world = comm.world_size
    cfg = EmbeddingCollectionConfig()
    t = table(kind, cap=cap, weight_dtype=wdtype, **kw)
    names = [f"k{i}" for i in range(lookups)]
    cfg.embedding_lookup([t] * lookups, names, "emb", ["sum"] * lookups)
    cfg.shard([["t"] for _ in range(world)], [("mp", ["t"])])
    return EmbeddingCollection(cfg, b, {n: H for n in names}, comm.device, torch.float32, comm,
                               opt or CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1), seed=seed,
                               key_dtype=key_dtype, weighted=weighted)


def train_step(e, keys, weights=None, lr=0.05):
    """one training step on this rank's keys; returns the pooled outputs before the update"""
    dev = e.device
    e.set_keys(torch.as_tensor(keys, dtype=torch.int64).to(dev))
    if weights is not None:
        e.set_weights(torch.as_tensor(weights, dtype=torch.float32).to(dev))
    e.forward(True)
    out = e.top_data["emb"].clone()
    g = e.top_grad["emb"]
    g.copy_((0.5 * e.top_data["emb"] + 0.01).to(g.dtype))
    e.backward(torch.tensor([lr], device=dev), torch.tensor([1], dtype=torch.int32, device=dev))
    return out


def by_key(e, name="t"):
    """{key: (weights, states)} of every row held here"""
    res = {}
    for (k, w, _, sts, _) in e.dump_table_local(name):
        for i, key in enumerate(k.tolist()):
            res[key] = (w[i], [None if s is None else s[i] for s in sts])
    return res


def assert_same_tables(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert torch.equal(a[k][0], b[k][0]), k
        for x, y in zip(a[k][1], b[k][1]):
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), k


class AdmitModel:
    """plain-Python admission: exact counts per key (halved when the clock is a multiple of P), one step =
    tick, decay, count every occurrence of a key without a row, then blank (-1) every position of a missing
    key whose count is below the threshold.  ``present`` is told after the step which keys have rows."""

    def __init__(self, threshold, period=0):
        self.thr, self.P = threshold, period
        self.counts, self.clock = {}, 0
        self.counted = self.rejected = 0

    def filter(self, lookups, present):
        self.clock += 1
        if self.P and self.clock % self.P == 0:
            self.counts = {k: c // 2 for k, c in self.counts.items()}
        for keys in lookups:
            for k in keys:
                if k >= 0 and k not in present:
                    self.counts[k] = self.counts.get(k, 0) + 1
                    self.counted += 1
        out = []
        for keys in lookups:
            row = []
            for k in keys:
                rej = k >= 0 and k not in present and self.counts.get(k, 0) < self.thr
                self.rejected += rej
                row.append(-1 if rej else k)
            out.append(row)
        return out


def collision_free(keys, width):
    """every key has a sketch row in which no other key of ``keys`` shares its counter: then every minimum
    equals the key's exact count, and no decision depends on a collision"""
    keys = sorted(set(int(k) for k in keys if k >= 0))
    sl = sketch_slots(keys, width)
    ok = np.zeros(len(keys), dtype=bool)
    for r in range(4):
        _, inv, cnt = np.unique(sl[:, r], return_inverse=True, return_counts=True)
        ok |= cnt[inv] == 1
    return bool(ok.all())


# ----------------------------------------------------------------------------- validation
def test_admit_options_validation():
    for bad in (2.0, "2", True, None):
        with pytest.raises(ValueError, match="table a.*admit_threshold must be an int"):
            EmbeddingTableConfig("a", -1, 8, admit_threshold=bad)
        with pytest.raises(ValueError, match="table a.*admit_decay_steps must be an int"):
            EmbeddingTableConfig("a", -1, 8, admit_threshold=2, admit_decay_steps=bad)
    for bad in (0, -1, 1 << 32):
        with pytest.raises(ValueError, match="table b.*admit_threshold"):
            EmbeddingTableConfig("b", -1, 8, admit_threshold=bad)
    with pytest.raises(ValueError, match="table b.*admit_decay_steps"):
        EmbeddingTableConfig("b", -1, 8, admit_threshold=2, admit_decay_steps=-1)
    with pytest.raises(ValueError, match="table c.*admit_threshold needs a dynamic table"):
        EmbeddingTableConfig("c", 100, 8, admit_threshold=2)
    with pytest.raises(ValueError, match="table c.*admit_decay_steps needs a dynamic table"):
        EmbeddingTableConfig("c", 100, 8, admit_decay_steps=0)
    with pytest.raises(ValueError, match="table d.*admit_decay_steps needs admit_threshold > 1"):
        EmbeddingTableConfig("d", -1, 8, admit_decay_steps=4)
    t = EmbeddingTableConfig("e", -1, 8, max_capacity=64, evict_strategy="lru", admit_threshold=np.int64(3),
                             admit_decay_steps=5)
    assert (t.admit_threshold, t.admit_decay_steps) == (3, 5) and type(t.admit_threshold) is int
    d = EmbeddingTableConfig("f", -1, 8)
    assert (d.admit_threshold, d.admit_decay_steps) == (1, 0)


def test_admitting_placement_validation():
    """(an evicting table refuses these placements already, admitting or not)"""
    kind = "growing"
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(table(kind, cap=64, admit_threshold=2), "k", "emb", "sum")
    cfg.shard([["t"]], [("dp", ["t"])])
    with pytest.raises(ValueError, match="table t: an admitting table .*'dp'"):
        EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, Comm.single(CPU), CreateOptimizer(Optimizer_t.SGD))
    from hugectr_b200.parallel.emu import run_ranks

    def make(plan):
        cfg = EmbeddingCollectionConfig()
        cfg.embedding_lookup(table(kind, cap=64, admit_threshold=2), "k", "emb", "sum")
        cfg.shard(*plan)
        return run_ranks(2, lambda comm: EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, comm,
                                                              CreateOptimizer(Optimizer_t.SGD)) and True,
                         device=CPU, p2p=False)
    with pytest.raises(RuntimeError, match="table t: an admitting table .*column factor 2"):
        make(([["t"], ["t"]], [("mp", [("t", 2)])]))
    assert make(([["t"], ["t"]], [("mp", ["t"])])) == [True, True]          # row-wise: accepted


# ----------------------------------------------------------------------------- graph JSON
def _json_model(**kw):
    solver = hugectr.CreateSolver(batchsize=16, batchsize_eval=16, lr=0.01, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic"], eval_source="synthetic",
                                  check_type=hugectr.Check_t.Non, slot_size_array=[100, 100])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("a", 2, False, 1),
                                                        hugectr.DataReaderSparseParam("b", 1, True, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup([hugectr.EmbeddingTableConfig("dyn", -1, 8, init_capacity=77, **kw),
                          hugectr.EmbeddingTableConfig("st", 100, 8)], ["a", "b"], "emb", ["sum", "sum"])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["c"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    return m, rp


@pytest.mark.parametrize("kw", [dict(admit_threshold=3), dict(admit_threshold=2, admit_decay_steps=7),
                                dict(admit_threshold=4, max_capacity=96, evict_strategy="lfu")])
def test_graph_json_round_trips_the_admit_options(tmp_path, kw):
    m, rp = _json_model(**kw)
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    tj = {t["name"]: t for t in [l for l in json.load(open(p))["layers"] if l["type"] == "EmbeddingCollection"][0]["tables"]}
    assert tj["dyn"]["admit_threshold"] == kw["admit_threshold"]
    assert tj["dyn"].get("admit_decay_steps") == kw.get("admit_decay_steps")
    assert "admit_threshold" not in tj["st"] and "admit_decay_steps" not in tj["st"]
    m2 = hugectr.Model(hugectr.CreateSolver(batchsize=16, batchsize_eval=16, lr=0.01, vvgpu=[[0]], use_cuda_graph=False),
                       rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m2.construct_from_json(p)
    m2.compile()
    t = {x.name: x for x in m2.ebc_configs[0].tables()}
    assert (t["dyn"].admit_threshold, t["dyn"].admit_decay_steps) == (kw["admit_threshold"], kw.get("admit_decay_steps", 0))
    p2 = str(tmp_path / "g2.json")
    m2.graph_to_json(p2)
    assert open(p, "rb").read() == open(p2, "rb").read()


def test_graph_json_without_admit_options_has_no_such_keys(tmp_path):
    m, _ = _json_model()
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    assert b"admit_" not in open(p, "rb").read()


# ----------------------------------------------------------------------------- the rules by hand
@pytest.mark.parametrize("kind", KINDS)
def test_rules_by_hand_threshold_3(kind):
    b, K, Q, R = 4, 10**12 + 7, 10**12 + 99, 5
    e = collection(Comm.single(CPU), kind, b, 1, lookups=1, opt=CreateOptimizer(Optimizer_t.SGD),
                   admit_threshold=3)
    ev = e.eval_clone(b)
    sk = e._admit_sketches()[0]
    st = lambda: e.admission_stats()[("t", 0)]
    mins = lambda k: int(sk.values().view(-1)[torch.from_numpy(sketch_slots([k], sk.width)[0])].min())
    # step 1: two occurrences of K are rejected: they read zero, get no row and no update
    out = train_step(e, [K, K, -1, -1])
    assert bool((out[:2] == 0).all()) and st() == {"counted": 2, "rejected": 2} and by_key(e) == {}
    # an evaluation lookup changes nothing (no count, no insert, no tick)
    before, clock = sk.values().clone(), int(e.evict_clock[0])
    ev.set_keys(torch.tensor([K, R, R, R]))
    ev.forward(False)
    assert torch.equal(sk.values(), before) and int(e.evict_clock[0]) == clock and st()["counted"] == 2
    assert bool((ev.top_data["emb"] == 0).all())
    # step 2: a third occurrence admits K
    out = train_step(e, [K, -1, -1, -1])
    assert bool((out[0] != 0).any()) and st() == {"counted": 3, "rejected": 2} and sorted(by_key(e)) == [K]
    # step 3: three occurrences of Q admit it in the same step; K has a row and does not count
    out = train_step(e, [Q, Q, Q, K])
    assert bool((out != 0).any(1).all()) and st() == {"counted": 6, "rejected": 2}
    assert sorted(by_key(e)) == sorted([K, Q]) and mins(K) == 3 and mins(Q) == 3


@pytest.mark.parametrize("kind", ["growing", "lfu"])
def test_decay_halves_the_counts_at_the_right_clock(kind):
    b, K = 4, 12345
    e = collection(Comm.single(CPU), kind, b, 1, lookups=1, admit_threshold=3, admit_decay_steps=2)
    sk = e._admit_sketches()[0]
    cnt = lambda: [int(x) for x in sk.values().view(-1)[torch.from_numpy(sketch_slots([K], sk.width)[0])]]
    train_step(e, [K, K, K, -1])                       # clock 1: counted to 3, admitted
    assert cnt() == [3] * 4 and int(sk.values().sum()) == 12
    train_step(e, [-1] * 4)                            # clock 2: halved to 1
    assert cnt() == [1] * 4
    train_step(e, [-1] * 4)                            # clock 3: no decay
    assert cnt() == [1] * 4
    train_step(e, [-1] * 4)                            # clock 4: 0
    assert cnt() == [0] * 4


def test_counters_saturate():
    sk = AdmitSketch(100, 2, 0, torch.zeros(1, dtype=torch.int64), CPU)
    sl = torch.from_numpy(sketch_slots([77], sk.width)[0])
    sk.counters[sl] = torch.tensor([-3, -2, -1, 5], dtype=torch.int32)        # 2**32 - 3, - 2, - 1, 5
    sk.count([77] * 10)
    assert sk.values().view(-1)[sl].tolist() == [(1 << 32) - 1] * 3 + [15]


# ----------------------------------------------------------------------------- against the model of the rules
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
@pytest.mark.parametrize("period", [0, 3])
def test_collection_matches_the_model_of_the_rules(kind, opt, period):
    """threshold 2: outputs, rows, weights and state equal those of the same table without admission fed the
    stream with the positions the model of the rules rejects blanked, after every step; the counters equal
    the model's (the key set is collision-free in the sketch)"""
    b, H, cap = 16, 2, 256 if kind == "growing" else 32
    o = CreateOptimizer(Optimizer_t.SGD) if opt == "sgd" else CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1)
    batches = power_law_batches(12, 1, 2 * b * H, 400, seed=5)
    ea = collection(Comm.single(CPU), kind, b, H, cap=cap, opt=o, admit_threshold=2, admit_decay_steps=period)
    ep = collection(Comm.single(CPU), kind, b, H, cap=cap, opt=o)
    assert collision_free(np.concatenate([k[0] for k in batches]), ea._admit_sketches()[0].width)
    model = AdmitModel(2, period)
    for keys in batches:
        present = set(by_key(ep))
        filt = model.filter([list(keys[0][:b * H]), list(keys[0][b * H:])], present)
        oa = train_step(ea, keys[0])
        op = train_step(ep, np.array(filt[0] + filt[1]))
        assert torch.equal(oa, op)
        assert_same_tables(by_key(ea), by_key(ep))
        assert ea.admission_stats()[("t", 0)] == {"counted": model.counted, "rejected": model.rejected}
    assert model.rejected > 0 and len(by_key(ea)) > 0
    if kind != "growing":
        assert ea.eviction_stats()[("t", 0)]["evicted"] > 0


@pytest.mark.parametrize("kind", KINDS)
def test_threshold_1_is_bit_identical_to_no_option(kind):
    b, H = 16, 2
    batches = power_law_batches(8, 1, 2 * b * H, 400, seed=6)
    e1 = collection(Comm.single(CPU), kind, b, H, cap=128, admit_threshold=1)
    e0 = collection(Comm.single(CPU), kind, b, H, cap=128)
    for keys in batches:
        assert torch.equal(train_step(e1, keys[0]), train_step(e0, keys[0]))
    assert_same_tables(by_key(e1), by_key(e0))
    assert e1.admission_stats() == {} and e1._admit_sketches() == [] and e1.memory_bytes() == e0.memory_bytes()
    assert e1.eviction_stats() == e0.eviction_stats()


def test_memory_bytes_counts_the_sketch():
    e1 = collection(Comm.single(CPU), "lru", 4, 1, cap=393_216, lookups=1, admit_threshold=2)
    e0 = collection(Comm.single(CPU), "lru", 4, 1, cap=393_216, lookups=1)
    assert e1.memory_bytes() - e0.memory_bytes() == 16 << 20          # 4 x 2**20 uint32 counters
    assert e1._admit_sketches()[0].width == 1 << 20


# ----------------------------------------------------------------------------- emulated ranks, row-sharded
def shard_oracle(batches, world, kind, cap, b, H, thr, period):
    """per-step live keys and final counters of every shard: one CPU table (+ sketch) per shard fed the keys of
    every rank, the rules applied by hand in the order of the collection"""
    from hugectr_b200.embedding.hashtable import HashTable, SetAssocTable
    clock = torch.zeros(1, dtype=torch.int64)
    tabs = []
    for s in range(world):
        sk = AdmitSketch((cap + 31) // 32 * 32 if kind != "growing" else cap, thr, period, clock, CPU)
        if kind == "growing":
            t = HashTable(cap, CPU)
            t.sketch = sk
        else:
            t = SetAssocTable(cap, kind, clock, CPU, sketch=sk)
        tabs.append(t)
    res = []
    for keys in batches:
        clock.add_(1)
        for t in tabs:
            t.sketch.decay()
        for s, t in enumerate(tabs):
            regs = [torch.tensor(np.stack([kb[l * b * H:(l + 1) * b * H] for kb in keys])) for l in range(2)]
            if kind == "growing":
                ks = [torch.where((r >= 0) & (r % world == s), r, torch.full_like(r, -1)).reshape(-1) for r in regs]
                for k in ks:
                    t.admit_count(k)
                for k in ks:
                    t.admit_filter(k)
                    t.get_insert(k)
            else:
                for r in regs:
                    t.touch(r, 0, r.shape[1], world, s)
                for r in regs:
                    t.insert(r, 0, r.shape[1], world, s)
        res.append([sorted(t.dump()[0].tolist()) for t in tabs])
    return res, [t.sketch for t in tabs]


def _shard_run(comm, kind, batches, cap, b, H, thr, period):
    e = collection(comm, kind, b, H, cap=cap, admit_threshold=thr, admit_decay_steps=period)
    lives = []
    for keys in batches:
        train_step(e, keys[comm.rank])
        lives.append(sorted(k for k in by_key(e)))
    return lives, e.admission_stats(), e._admit_sketches()[0].values(), e.fused


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_emulated_ranks_row_sharded_match_the_oracle(world, kind):
    from hugectr_b200.parallel.emu import run_ranks
    b, H, cap, steps = 8, 2, 64, 8
    batches = power_law_batches(steps, world, 2 * b * H, 300, seed=world)
    res = run_ranks(world, lambda comm: _shard_run(comm, kind, batches, cap, b, H, 2, 3), device=CPU, p2p=False)
    ref, sks = shard_oracle(batches, world, kind, cap, b, H, 2, 3)
    for s in range(world):
        for step in range(steps):
            assert res[s][0][step] == ref[step][s], (step, s)
        assert torch.equal(res[s][2], sks[s].values())
        assert res[s][1][("t", s)] == dict(zip(("counted", "rejected"), sks[s].stats.tolist()))
    if kind != "growing":
        return
    # collision-free keys: the admitted set does not depend on the plan (one process, same keys)
    allk = np.concatenate([kb for keys in batches for kb in keys])
    assert collision_free(allk, 1024)
    one = [[np.concatenate([keys[r][l * b * H:(l + 1) * b * H] for r in range(world)]) for l in range(2)]
           for keys in batches]
    e = collection(Comm.single(CPU), kind, world * b, H, cap=world * cap, admit_threshold=2, admit_decay_steps=3)
    assert e._admit_sketches()[0].width == 1024
    for step, keys in enumerate(one):
        train_step(e, np.concatenate(keys))
        assert sorted(by_key(e)) == sorted(k for s in range(world) for k in ref[step][s]), step


# ----------------------------------------------------------------------------- checkpoints
@pytest.mark.parametrize("kind", KINDS)
def test_checkpoint_round_trip_admitted_keys_only(kind):
    b, H = 16, 2
    batches = power_law_batches(6, 1, 2 * b * H, 400, seed=8)
    e = collection(Comm.single(CPU), kind, b, H, cap=128, admit_threshold=3)
    for keys in batches:
        train_step(e, keys[0])
    (k, w, _, sts, _), = e.dump_table_local("t")
    stream = np.concatenate([x[0] for x in batches])
    seen = {int(x): int((stream == x).sum()) for x in np.unique(stream)}
    assert len(k) and set(k.tolist()) < set(seen) and all(seen[x] >= 3 for x in k.tolist())
    assert e.admission_stats()[("t", 0)]["rejected"] > 0
    e2 = collection(Comm.single(CPU), kind, b, H, cap=128, admit_threshold=3, seed=99)
    e2.load_table_rows("t", k, w, sts)
    assert_same_tables(by_key(e2), by_key(e))                # every key loaded, none counted
    assert e2.admission_stats()[("t", 0)] == {"counted": 0, "rejected": 0}
    assert int(e2._admit_sketches()[0].values().sum()) == 0


# ----------------------------------------------------------------------------- weighted inputs
@pytest.mark.parametrize("kind", ["growing", "lru"])
def test_weighted_input_counts_occurrences_not_weights(kind):
    b, K = 4, 4242
    e = collection(Comm.single(CPU), kind, b, 1, lookups=1, weighted=("k0",), admit_threshold=3)
    out = train_step(e, [K, K, -1, -1], weights=[5.0, 5.0, 1.0, 1.0])
    assert e.admission_stats()[("t", 0)] == {"counted": 2, "rejected": 2} and bool((out == 0).all())
    out = train_step(e, [K, -1, -1, -1], weights=[0.5, 1.0, 1.0, 1.0])
    assert sorted(by_key(e)) == [K] and bool((out[0] != 0).any())


# ----------------------------------------------------------------------------- Model.fit
def _fit_model(kind, device=CPU, cap=64, **kw):
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]], repeat_dataset=True,
                                  max_eval_batches=2, use_cuda_graph=device.type == "cuda")
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"],
                                  eval_source="synthetic:1.0", check_type=hugectr.Check_t.Non, slot_size_array=[5000])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad), comm=Comm.single(device))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("k", 2, False, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig()
    ebc.embedding_lookup(table(kind, cap=cap, **kw), "k", "emb", "sum")
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=8))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    return m


@pytest.mark.parametrize("kind", ["growing", "lru"])
def test_model_fit_logs_the_admission_counters(kind, monkeypatch):
    from hugectr_b200.utils import logger
    said = []
    real = logger.info
    monkeypatch.setattr(logger, "info", lambda msg, *a, **k: (said.append(str(msg)), real(msg, *a, **k)))
    m = _fit_model(kind, cap=8192 if kind == "growing" else 64, admit_threshold=2, admit_decay_steps=10)
    m.fit(max_iter=30, display=10, eval_interval=15, snapshot=10**9)
    st = m.ebcs_train[0].admission_stats()[("t", 0)]
    assert st["counted"] > 0 and st["rejected"] > 0
    lines = [x for x in said if x.startswith("admitting embedding table t shard 0")]
    assert len(lines) >= 3 and lines[-1].endswith(f"counted {st['counted']} rejected {st['rejected']}")
    assert m.get_current_loss() == m.get_current_loss()
