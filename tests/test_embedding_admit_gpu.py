"""Admission of new keys to dynamic tables on the H100: the kernels against the CPU sketch and tables, one key at
10 000 positions, training against the CPU path, threshold 1 against no option, one CUDA-graph capture with the
decay inside the replays, and emulated ranks on the peer-memory path."""
import pytest
import torch

from hugectr_b200.embedding.hashtable import AdmitSketch, HashTable, SetAssocTable, sketch_slots
from hugectr_b200.enums import Optimizer_t
from hugectr_b200.ops import dense as D
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

from test_embedding_admit_cpu import _fit_model, _shard_run, by_key, collection, shard_oracle, train_step
from test_embedding_evict_cpu import power_law_batches

pytestmark = pytest.mark.gpu
CPU, DEV = torch.device("cpu"), torch.device("cuda")


def make(kind, cap, dev, clock, thr, period):
    sk = AdmitSketch(cap, thr, period, clock, dev)
    if kind == "growing":
        t = HashTable(cap, dev)
        t.sketch = sk
        return t
    return SetAssocTable(cap, kind, clock, dev, sketch=sk)


def step(t, regions, kind):
    """one training lookup of a table over the key regions ([1, n] each, rows written in place)"""
    t.sketch.clock.add_(1)          # (an evicting table shares its clock with its sketch)
    t.sketch.decay()
    if kind == "growing":
        ks = [r.view(-1).to(torch.int64) for r in regions]
        for k in ks:
            t.admit_count(k)
        for r, k in zip(regions, ks):
            t.admit_filter(k)
            r.view(-1).copy_(t.get_insert(k).to(r.dtype))
        return
    for r in regions:
        t.touch(r, 0, r.shape[1])
    for r in regions:
        t.insert(r, 0, r.shape[1])


@pytest.mark.parametrize("kind,key_dtype", [("lru", torch.int64), ("lfu", torch.int64), ("lru", torch.int32),
                                            ("lfu", torch.int32), ("growing", torch.int64)])
def test_kernels_match_the_cpu_sketch_and_table(kind, key_dtype):
    """40 power-law batches of two lookups, threshold 2, decay every 4 steps: the counters, the counted and
    rejected totals, the rejected positions and the table (live keys with stamps and counts, the eviction
    counters) equal the CPU implementation's after every step"""
    n, steps = 512, 40
    cap = 16384 if kind == "growing" else 2048          # (a growing table that never runs out of rows)
    gclock, cclock = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64)
    g, c = make(kind, cap, DEV, gclock, 2, 4), make(kind, cap, CPU, cclock, 2, 4)
    assert g.sketch.width == c.sketch.width == 2 * cap
    batches = power_law_batches(steps, 1, 2 * n, 30000, seed=3)
    mask = (1 << 31) - 1 if key_dtype == torch.int32 else (1 << 62) - 1
    for keys in batches:
        kk = torch.as_tensor(keys[0] & mask).view(2, n)
        gb, cb = kk.to(DEV, key_dtype).contiguous(), kk.clone()
        step(g, [gb[0:1], gb[1:2]], kind)
        step(c, [cb[0:1], cb[1:2]], kind)
        assert torch.equal(g.sketch.values(), c.sketch.values())
        assert torch.equal(g.sketch.stats.cpu(), c.sketch.stats)
        assert torch.equal(gb.cpu() < 0, cb < 0)
        if kind == "growing":
            assert sorted(g.dump()[0].tolist()) == sorted(c.dump()[0].tolist())
            continue
        gk, gs = g.dump()
        ck, cs = c.dump()
        assert torch.equal(gk, ck)
        s = gs.to(DEV)
        assert g.stamps[s].cpu().tolist() == c.stamps[cs].tolist() and g.counts[s].cpu().tolist() == c.counts[cs].tolist()
        assert torch.equal(g.stats.cpu(), c.stats)
        rows = gb.long()
        ok = rows >= 0
        assert torch.equal(g.keys[rows[ok]].cpu(), kk[ok.cpu()].long())
    st = c.sketch.stats.tolist()
    assert st[0] > 0 and st[1] > 0


@pytest.mark.parametrize("kind", ["lru", "growing"])
def test_one_key_at_10000_positions(kind):
    n, K = 10_000, 987_654_321_012
    for thr, admitted in ((10_000, True), (10_001, False)):
        t = make(kind, 1024, DEV, torch.zeros(1, dtype=torch.int64, device=DEV), thr, 0)
        buf = torch.full((1, n), K, dtype=torch.int64, device=DEV)
        step(t, [buf], kind)
        sl = torch.from_numpy(sketch_slots([K], t.sketch.width)[0])
        assert t.sketch.values().view(-1)[sl].tolist() == [n] * 4
        assert t.sketch.stats.cpu().tolist() == [n, 0 if admitted else n]
        rows = buf.view(-1).cpu()
        if admitted:
            assert bool((rows == rows[0]).all()) and int(rows[0]) >= 0
        else:
            assert bool((rows == -1).all())
        assert sorted(t.dump()[0].tolist()) == ([K] if admitted else [])


def test_counters_saturate_on_the_device():
    clock = torch.zeros(1, dtype=torch.int64, device=DEV)
    t = make("lru", 64, DEV, clock, 2, 0)
    sl = torch.from_numpy(sketch_slots([77], t.sketch.width)[0]).to(DEV)
    t.sketch.counters[sl] = torch.tensor([-3, -2, -1, 5], dtype=torch.int32, device=DEV)
    step(t, [torch.full((1, 1000), 77, dtype=torch.int64, device=DEV)], "lru")
    assert t.sketch.counters[sl].cpu().long().tolist() == [-1, -1, -1, 1005]


@pytest.mark.parametrize("kind", ["growing", "lfu"])
@pytest.mark.parametrize("arm", ["adagrad", "rowwise_adagrad", "bf16"])
def test_training_matches_the_cpu_path(kind, arm):
    """15 steps of a collection with one admitting table (threshold 2, decay 4; two lookups; int32 keys for the
    growing table): the live keys, counters and admission totals match the CPU path exactly after every step,
    the weights and state of the live keys by key within the tolerances of the eviction tests"""
    opt = CreateOptimizer(Optimizer_t.RowWiseAdaGrad if arm == "rowwise_adagrad" else Optimizer_t.AdaGrad,
                          initial_accu_value=0.1, epsilon=1e-7)
    wdt = "bf16" if arm == "bf16" else "fp32"
    b, H = 64, 2
    cap = 4096 if kind == "growing" else 128
    batches = power_law_batches(15, 1, 2 * b * H, 4000, seed=9)
    kdt = torch.int32 if kind == "growing" else torch.int64
    if kdt == torch.int32:
        batches = [[k & ((1 << 31) - 1) for k in x] for x in batches]
    eg = collection(Comm.single(DEV), kind, b, H, cap=cap, opt=opt, wdtype=wdt, admit_threshold=2,
                    admit_decay_steps=4, key_dtype=kdt)
    ec = collection(Comm.single(CPU), kind, b, H, cap=cap, opt=opt, wdtype=wdt, admit_threshold=2,
                    admit_decay_steps=4, key_dtype=kdt)
    if kind == "growing":
        # a growing table initialises by row, and the device hands out rows in the order its inserts race:
        # one initial value for every row makes the weights comparable by key
        for e in (eg, ec):
            for grp in e.groups:
                grp.table.fill_(0.01)
    for keys in batches:
        train_step(eg, keys[0])
        train_step(ec, keys[0])
        assert sorted(by_key(eg)) == sorted(by_key(ec))
        assert eg.admission_stats() == ec.admission_stats()
        assert torch.equal(eg._admit_sketches()[0].values(), ec._admit_sketches()[0].values())
    assert eg.admission_stats()[("t", 0)]["rejected"] > 0
    if kind != "growing":
        assert eg.eviction_stats()[("t", 0)]["evicted"] > 0
    (kg, wg, _, sg, _), = eg.dump_table_local("t")
    (kc, wc, _, sc, _), = ec.dump_table_local("t")
    assert torch.equal(kg, kc) and len(kg) > 0
    tol = dict(rtol=2e-2, atol=2e-3) if wdt == "bf16" else dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(wg, wc, **tol)
    torch.testing.assert_close(sg[0], sc[0], **(dict(rtol=1e-2, atol=1e-3) if wdt == "bf16" else tol))


@pytest.mark.parametrize("kind", ["growing", "lru", "lfu"])
def test_threshold_1_is_bit_identical_on_the_device(kind):
    """no sketch and the same launches every step; the same live keys and eviction counters.  Outputs and weights
    agree to rounding only: which way or row a key takes depends on the order its warps race in, with or without
    the option, and the backward sums a row's gradients in arena order"""
    b, H = 64, 2
    batches = power_law_batches(8, 1, 2 * b * H, 3000, seed=6)
    e1 = collection(Comm.single(DEV), kind, b, H, cap=512, admit_threshold=1)
    e0 = collection(Comm.single(DEV), kind, b, H, cap=512)
    assert e1._admit_sketches() == [] and e1.memory_bytes() == e0.memory_bytes()
    for keys in batches:
        n0 = D.launch_count
        o1 = train_step(e1, keys[0])
        n1 = D.launch_count
        o0 = train_step(e0, keys[0])
        assert D.launch_count - n1 == n1 - n0
        if kind != "growing":
            torch.testing.assert_close(o1, o0, rtol=1e-5, atol=1e-7)
        assert sorted(by_key(e1)) == sorted(by_key(e0))
    if kind != "growing":
        t1, t0 = by_key(e1), by_key(e0)
        for k in t1:
            torch.testing.assert_close(t1[k][0], t0[k][0], rtol=1e-5, atol=1e-7)
        assert e1.eviction_stats() == e0.eviction_stats()
    assert e1.admission_stats() == {}


@pytest.mark.parametrize("kind", ["growing", "lru"])
def test_model_fit_captures_the_step_graph_once_and_decays_in_the_replays(kind, monkeypatch):
    import torch.cuda as tc
    made = []

    class Counting(tc.CUDAGraph):
        def __init__(self, *a, **k):
            made.append(1)
            super().__init__(*a, **k)
    monkeypatch.setattr(tc, "CUDAGraph", Counting)
    m = _fit_model(kind, device=DEV, cap=8192 if kind == "growing" else 64, admit_threshold=2, admit_decay_steps=5)
    m.fit(max_iter=60, display=10, eval_interval=0, snapshot=10**9)
    e = m.ebcs_train[0]
    st = e.admission_stats()[("t", 0)]
    assert st["counted"] > 0 and st["rejected"] > 0
    assert m._graph is not None and len(made) == 1
    assert int(e.evict_clock[0]) == 60
    # without decay the four rows would hold exactly 4 * counted (nothing saturates here)
    assert int(e._admit_sketches()[0].values().sum()) < 4 * st["counted"]


@pytest.mark.parametrize("kind", ["growing", "lru", "lfu"])
def test_emulated_ranks_peer_memory_path_matches_the_oracle(kind):
    from hugectr_b200.parallel.emu import run_ranks
    world, b, H, cap, steps = 4, 32, 2, 512, 10
    batches = power_law_batches(steps, world, 2 * b * H, 20000, seed=4)

    res = run_ranks(world, lambda comm: _shard_run(comm, kind, batches, cap, b, H, 2, 3), device=DEV)
    ref, sks = shard_oracle(batches, world, kind, cap, b, H, 2, 3)
    for s in range(world):
        assert res[s][3]                                 # the peer-memory path
        for st in range(steps):
            assert res[s][0][st] == ref[st][s], (st, s)
        assert torch.equal(res[s][2], sks[s].values())
        assert res[s][1][("t", s)] == dict(zip(("counted", "rejected"), sks[s].stats.tolist()))
