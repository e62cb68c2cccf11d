"""Evicting dynamic tables (EmbeddingTableConfig(evict_strategy="lru" | "lfu")) on the CPU path: validation,
graph JSON, the CPU table against an independent model of the rules, Model.fit past the point where a growing
table stops, row-sharded emulated ranks and the checkpoint round trip."""
import json

import numpy as np
import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                               EmbeddingTableConfig)
from hugectr_b200.embedding.hashtable import SetAssocTable, evict_set_of
from hugectr_b200.enums import Optimizer_t
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

CPU = torch.device("cpu")


# ----------------------------------------------------------------------------- an independent model of the rules
class RuleModel:
    """sets of at most 32 keys, each key with (stamp, count); one step = touch every present key of every
    lookup, then insert the missing keys in stream order"""

    def __init__(self, num_sets, strategy):
        self.S, self.lfu = num_sets, strategy == "lfu"
        self.sets = [dict() for _ in range(num_sets)]
        self.clock = 0
        self.dropped = self.evicted = 0

    def step(self, lookups):
        self.clock += 1
        now = self.clock
        for keys in lookups:
            for k in keys:
                d = self.sets[int(evict_set_of([k], self.S)[0])]
                if k in d:
                    st, c = d[k]
                    d[k] = (now, c + 1)
        for keys in lookups:
            for k in keys:
                d = self.sets[int(evict_set_of([k], self.S)[0])]
                if k in d:
                    continue
                if len(d) == 32:
                    cand = [x for x, (st, _) in d.items() if st != now]
                    if not cand:
                        self.dropped += 1
                        continue
                    v = min(cand, key=lambda x: ((min(d[x][1], (1 << 32) - 1) if self.lfu else 0), d[x][0], x))
                    del d[v]
                    self.evicted += 1
                d[k] = (now, 1)

    def state(self):
        return {k: v for d in self.sets for k, v in d.items()}


def table_state(t):
    keys, slots = t.dump()
    return {int(k): (int(t.stamps[s]), int(t.counts[s])) for k, s in zip(keys.tolist(), slots.tolist())}


def run_table(t, lookups):
    """one training lookup of the CPU table over the key lists ``lookups``; returns the rows"""
    t.clock.add_(1)
    bufs = [torch.tensor(k, dtype=torch.int64).view(1, -1) for k in lookups]
    for b in bufs:
        t.touch(b, 0, b.shape[1])
    for b in bufs:
        t.insert(b, 0, b.shape[1])
    return [b.view(-1).tolist() for b in bufs]


def keys_of_set(s, num_sets, n, start=1):
    out, k = [], start
    while len(out) < n:
        if int(evict_set_of([k], num_sets)[0]) == s:
            out.append(k)
        k += 1
    return out


# ----------------------------------------------------------------------------- validation
def test_evict_strategy_validation():
    with pytest.raises(ValueError, match="table a.*evict_strategy"):
        EmbeddingTableConfig("a", -1, 8, max_capacity=64, evict_strategy="fifo")
    with pytest.raises(ValueError, match="table b.*dynamic"):
        EmbeddingTableConfig("b", 100, 8, max_capacity=64, evict_strategy="lru")
    with pytest.raises(ValueError, match="table c.*max_capacity"):
        EmbeddingTableConfig("c", -1, 8, evict_strategy="lfu")
    assert EmbeddingTableConfig("d", -1, 8).evict_strategy is None

    def collection(plan, world=2):
        cfg = EmbeddingCollectionConfig()
        cfg.embedding_lookup(EmbeddingTableConfig("t", -1, 8, max_capacity=64, evict_strategy="lru"), "k", "emb", "sum")
        cfg.shard(*plan)
        from hugectr_b200.parallel.emu import run_ranks
        return run_ranks(world, lambda comm: EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, comm,
                                                                  CreateOptimizer(Optimizer_t.SGD)), device=CPU, p2p=False)
    with pytest.raises(RuntimeError, match="table t.*'dp'"):
        collection(([["t"], ["t"]], [("dp", ["t"])]))
    with pytest.raises(RuntimeError, match="table t.*column factor 2"):
        collection(([["t"], ["t"]], [("mp", [("t", 2)])]))
    collection(([["t"], ["t"]], [("mp", ["t"])]))            # row-wise: accepted


def test_evict_strategy_validation_error_type_at_construction():
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(EmbeddingTableConfig("t", -1, 8, max_capacity=64, evict_strategy="lfu"), "k", "emb", "sum")
    cfg.shard([["t"]], [("dp", ["t"])])
    with pytest.raises(ValueError, match="table t"):
        EmbeddingCollection(cfg, 4, {"k": 1}, CPU, torch.float32, Comm.single(CPU), CreateOptimizer(Optimizer_t.SGD))


# ----------------------------------------------------------------------------- graph JSON
def _json_model(evict):
    solver = hugectr.CreateSolver(batchsize=16, batchsize_eval=16, lr=0.01, vvgpu=[[0]], use_cuda_graph=False)
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic"], eval_source="synthetic",
                                  check_type=hugectr.Check_t.Non, slot_size_array=[100, 100])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("a", 2, False, 1),
                                                        hugectr.DataReaderSparseParam("b", 1, True, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig()
    kw = dict(evict_strategy=evict) if evict else {}
    ebc.embedding_lookup([hugectr.EmbeddingTableConfig("dyn", -1, 8, init_capacity=77, max_capacity=96, **kw),
                          hugectr.EmbeddingTableConfig("st", 100, 8)], ["a", "b"], "emb", ["sum", "sum"])
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["emb", "dense"], ["c"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    return m, solver, rp


@pytest.mark.parametrize("strategy", ["lru", "lfu"])
def test_graph_json_round_trips_evict_strategy(tmp_path, strategy):
    m, solver, rp = _json_model(strategy)
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    tj = [l for l in json.load(open(p))["layers"] if l["type"] == "EmbeddingCollection"][0]["tables"]
    assert [t.get("evict_strategy") for t in tj] == [strategy, None]
    m2 = hugectr.Model(hugectr.CreateSolver(batchsize=16, batchsize_eval=16, lr=0.01, vvgpu=[[0]], use_cuda_graph=False),
                       rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.SGD), comm=Comm.single(CPU))
    m2.construct_from_json(p)
    m2.compile()
    t = {x.name: x for x in m2.ebc_configs[0].tables()}
    assert t["dyn"].evict_strategy == strategy and t["dyn"].max_capacity == 96 and t["st"].evict_strategy is None
    p2 = str(tmp_path / "g2.json")
    m2.graph_to_json(p2)
    assert open(p, "rb").read() == open(p2, "rb").read()


def test_graph_json_without_evict_strategy_has_no_such_key(tmp_path):
    m, _, _ = _json_model(None)
    p = str(tmp_path / "g.json")
    m.graph_to_json(p)
    assert b"evict_strategy" not in open(p, "rb").read()


# ----------------------------------------------------------------------------- the CPU table against the rule model
@pytest.mark.parametrize("strategy", ["lru", "lfu"])
def test_cpu_table_follows_the_rules_on_two_sets(strategy):
    S = 2
    t = SetAssocTable(S * 32, strategy, torch.zeros(1, dtype=torch.int64), CPU)
    ref = RuleModel(S, strategy)
    a = keys_of_set(0, S, 80)
    b = keys_of_set(1, S, 80, start=a[-1] + 1)

    def step(*lookups):
        rows = run_table(t, [list(x) for x in lookups])
        ref.step([list(x) for x in lookups])
        assert table_state(t) == ref.state()
        assert int(t.stats[1]) == ref.evicted and int(t.stats[2]) == ref.dropped
        return rows

    # empty ways first: 20 keys of set 0 land in ways 0..19 of set 0, in stream order
    rows = step(a[:20])
    assert rows == [[i for i in range(20)]]
    # duplicates of a new key in one step occupy one way; two lookups of the table see the same row
    rows = step([a[20], a[20], b[0]], [a[20], b[0]])
    assert rows[0][0] == rows[0][1] == rows[1][0] == 20 and rows[0][2] == rows[1][1] == 32
    # fill set 0 (32 ways) over steps with distinct counts: a[0..3] get touched a lot (LFU keeps them)
    step(a[21:32], a[:4] * 3)
    for i in range(3):
        step(a[:4])
    # set 0 is full; 6 new keys evict the 6 smallest unprotected ways
    st_before = table_state(t)
    step(a[32:38])
    gone = set(st_before) - set(table_state(t))
    assert len(gone) == 6
    if strategy == "lru":
        # the oldest stamps; among equal stamps the smallest keys
        order = sorted((v[0], k) for k, v in st_before.items() if int(evict_set_of([k], S)[0]) == 0)
        assert gone == {k for _, k in order[:6]}
    else:
        assert not (gone & set(a[:4]))
    # keys of the running step survive several lookups of the table, even when the set is overrun
    live0 = [k for k in table_state(t) if int(evict_set_of([k], S)[0]) == 0]
    keep = live0[:10]
    rows = step(keep, a[40:70], keep)          # 30 new keys, 22 unprotected ways: 8 dropped
    assert rows[0] == rows[2] and all(r >= 0 for r in rows[0])
    assert all(k in table_state(t) for k in keep)
    assert int(t.stats[2]) == 8 and sum(r < 0 for r in rows[1]) == 8
    # every way protected: the extra keys are dropped and counted
    protected = [k for k in table_state(t) if int(evict_set_of([k], S)[0]) == 0]
    assert len(protected) == 32
    rows = step(protected, a[70:75])
    assert rows[1] == [-1] * 5 and int(t.stats[2]) == 13


def test_cpu_table_breaks_ties_by_key():
    S = 2
    for strategy in ("lru", "lfu"):
        t = SetAssocTable(S * 32, strategy, torch.zeros(1, dtype=torch.int64), CPU)
        a = keys_of_set(1, S, 40)
        shuffled = list(np.random.default_rng(0).permutation(a[:32]).tolist())
        run_table(t, [shuffled])                  # 32 keys, same stamp and count
        run_table(t, [a[32:35]])
        assert set(table_state(t)) == set(a[3:35])  # the three smallest keys went


# ----------------------------------------------------------------------------- Model.fit on the CPU path
def _fit_model(evict, device=CPU):
    solver = hugectr.CreateSolver(batchsize=32, batchsize_eval=32, lr=0.05, vvgpu=[[0]], repeat_dataset=True,
                                  max_eval_batches=2, use_cuda_graph=device.type == "cuda")
    rp = hugectr.DataReaderParams(hugectr.DataReaderType_t.RawAsync, source=["synthetic:1.0"],
                                  eval_source="synthetic:1.0", check_type=hugectr.Check_t.Non, slot_size_array=[5000])
    m = hugectr.Model(solver, rp, hugectr.CreateOptimizer(hugectr.Optimizer_t.AdaGrad), comm=Comm.single(device))
    m.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=2, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("k", 2, False, 1)]))
    ebc = hugectr.EmbeddingCollectionConfig()
    kw = dict(evict_strategy=evict) if evict else {}
    ebc.embedding_lookup(hugectr.EmbeddingTableConfig("t", -1, 8, init_capacity=16, max_capacity=64, **kw),
                         "k", "emb", "sum")
    m.add(ebc)
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["emb"], ["r"], leading_dim=8))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["r", "dense"], ["c"]))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["c"], ["fc"], num_output=1))
    m.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc", "label"], ["loss"]))
    m.compile()
    return m


def test_model_fit_with_an_evicting_table_runs_past_max_capacity():
    with pytest.raises(RuntimeError, match="max_capacity"):
        _fit_model(None).fit(max_iter=60, display=5, eval_interval=30, snapshot=10**9)
    m = _fit_model("lru")
    m.fit(max_iter=60, display=5, eval_interval=30, snapshot=10**9)
    st = m.ebcs_train[0].eviction_stats()[("t", 0)]
    assert st["live"] == 64 and st["evicted"] > 0 and st["admitted"] == st["live"] + st["evicted"]
    assert m.ebcs_train[0].groups[0].rows == 64                  # never grew
    assert m.get_current_loss() == m.get_current_loss()


# ----------------------------------------------------------------------------- emulated ranks, row-sharded
def _train_collection(comm, strategy, batches, cap, b, H, opt=None, wdtype="fp32", seed=7, grads=None):
    """an evicting table row-sharded over every rank, two lookups of it; returns the collection"""
    world = comm.world_size
    cfg = EmbeddingCollectionConfig()
    t = EmbeddingTableConfig("t", -1, 8, init_capacity=1000, max_capacity=cap, evict_strategy=strategy,
                             weight_dtype=wdtype)
    cfg.embedding_lookup([t, t], ["k0", "k1"], "emb", ["sum", "sum"])
    cfg.shard([["t"] for _ in range(world)], [("mp", ["t"])])
    dev = comm.device
    e = EmbeddingCollection(cfg, b, {"k0": H, "k1": H}, dev, torch.float32, comm,
                            opt or CreateOptimizer(Optimizer_t.AdaGrad, initial_accu_value=0.1), seed=seed,
                            key_dtype=torch.int64)
    lr, st = torch.tensor([0.05], device=dev), torch.tensor([1], dtype=torch.int32, device=dev)
    lives = []
    for keys in batches:
        kb = keys[comm.rank]                         # this rank's batch: [2 * b * H]
        e.set_keys(torch.as_tensor(kb, dtype=torch.int64).to(dev))
        e.forward(True)
        g = e.top_grad["emb"]
        g.copy_((0.5 * e.top_data["emb"] + 0.01).to(g.dtype) if grads is None else grads)
        e.backward(lr, st)
        lives.append(sorted(e._dyn_tables[("t", 0, comm.rank if world > 1 else 0)].dump()[0].tolist()))
    return e, lives


def power_law_batches(steps, world, n, pool, seed=0, alpha=1.2):
    rng = np.random.default_rng(seed)
    ids = rng.permutation(pool).astype(np.int64) * 2654435761 % (1 << 40)       # scrambled ids
    p = 1.0 / np.arange(1, pool + 1) ** alpha
    p /= p.sum()
    return [[ids[rng.choice(pool, n, p=p)] for _ in range(world)] for _ in range(steps)]


def oracle_lives(batches, world, strategy, cap, b, H):
    """per-step live keys of every shard: one CPU table per shard fed the keys of every rank"""
    res = []
    tabs = [SetAssocTable(cap, strategy, torch.zeros(1, dtype=torch.int64), CPU) for _ in range(world)]
    for keys in batches:
        for s, t in enumerate(tabs):
            regs = [torch.tensor(np.stack([kb[l * b * H:(l + 1) * b * H] for kb in keys])) for l in range(2)]
            t.clock.add_(1)
            for r in regs:
                t.touch(r, 0, r.shape[1], world, s)
            for r in regs:
                t.insert(r, 0, r.shape[1], world, s)
        res.append([sorted(t.dump()[0].tolist()) for t in tabs])
    return res


@pytest.mark.parametrize("strategy", ["lru", "lfu"])
def test_emulated_ranks_row_sharded_evicting_table_matches_the_oracle_cpu(strategy):
    from hugectr_b200.parallel.emu import run_ranks
    world, b, H, cap = 2, 16, 2, 64
    batches = power_law_batches(8, world, 2 * b * H, 600)
    res = run_ranks(world, lambda comm: _train_collection(comm, strategy, batches, cap, b, H)[1], device=CPU, p2p=False)
    ref = oracle_lives(batches, world, strategy, cap, b, H)
    for step in range(len(batches)):
        for s in range(world):
            assert res[s][step] == ref[step][s], (step, s)
    assert sum(len(x) for x in ref[-1]) == world * cap


# ----------------------------------------------------------------------------- checkpoints
def test_checkpoint_round_trip_and_overfull_load_cpu():
    b, H, cap = 16, 2, 64
    batches = power_law_batches(6, 1, 2 * b * H, 400)
    e, lives = _train_collection(Comm.single(CPU), "lfu", batches, cap, b, H)
    (k, w, _, sts, _), = e.dump_table_local("t")
    assert k.tolist() == lives[-1] and len(k) == cap
    e2, _ = _train_collection(Comm.single(CPU), "lfu", [], cap, b, H, seed=99)
    e2.load_table_rows("t", k, w, sts)
    (k2, w2, _, sts2, _), = e2.dump_table_local("t")
    assert torch.equal(k2, k) and torch.equal(w2, w) and all((x is None) == (y is None) and (x is None or torch.equal(x, y)) for x, y in zip(sts2, sts))
    st = e2._dyn_tables[("t", 0, 0)]
    assert int(st.stamps[st.keys >= 0].max()) == 0 and int(st.counts[st.keys >= 0].min()) == 1
    # more keys of one set than it has ways
    e3, _ = _train_collection(Comm.single(CPU), "lfu", [], cap, b, H)
    many = torch.tensor(keys_of_set(0, cap // 32, 40, start=10**6))
    with pytest.raises(RuntimeError, match=r"table t: shard 0 .*8 of 40"):
        e3.load_table_rows("t", many, torch.zeros(40, 8))
