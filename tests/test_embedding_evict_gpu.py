"""Evicting dynamic tables on the H100: the kernels against the CPU table, the adversarial set, training against
the CPU path, one CUDA-graph capture for the whole fit, emulated ranks on the peer-memory path and checkpoints."""
import numpy as np
import pytest
import torch

from hugectr_b200.embedding import ops as E
from hugectr_b200.embedding.hashtable import SetAssocTable
from hugectr_b200.enums import Optimizer_t
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.solver import CreateOptimizer

from test_embedding_evict_cpu import (_fit_model, _train_collection, keys_of_set, oracle_lives,
                                      power_law_batches)

pytestmark = pytest.mark.gpu
CPU, DEV = torch.device("cpu"), torch.device("cuda")


def by_key(t):
    keys, slots = t.dump()
    s = slots.to(t.stamps.device)
    return keys.tolist(), t.stamps[s].cpu().tolist(), t.counts[s].cpu().long().tolist()


@pytest.mark.parametrize("strategy,key_dtype", [("lru", torch.int64), ("lfu", torch.int64), ("lru", torch.int32)])
def test_kernels_match_the_cpu_table(strategy, key_dtype):
    """50 power-law batches of two lookups, capacity well below the distinct keys: the live keys, their stamps
    and counts and the counters equal the CPU table's after every step; admitted rows equal the initializer
    mirror bit for bit (fp32 and bf16 arenas) and their state the initial values"""
    cap, n, steps = 2048, 512, 50
    g = SetAssocTable(cap, strategy, torch.zeros(1, dtype=torch.int64, device=DEV), DEV)
    c = SetAssocTable(cap, strategy, torch.zeros(1, dtype=torch.int64), CPU)
    batches = power_law_batches(steps, 1, 2 * n, 30000, seed=3)
    mask = (1 << 31) - 1 if key_dtype == torch.int32 else (1 << 62) - 1
    ev, key = 8, E.evict_init_key(11, 5)
    w32 = torch.zeros(cap, ev, device=DEV)
    wbf = torch.zeros(cap, ev, dtype=torch.bfloat16, device=DEV)
    s0, s1 = torch.full((cap, ev), 7.0, device=DEV), torch.full((cap, ev), 7.0, device=DEV)
    r0 = torch.full((cap,), 7.0, device=DEV)
    adm = (torch.zeros(2 * n, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV))
    total_adm = 0
    for keys in batches:
        kk = torch.as_tensor(keys[0] & mask).view(2, n)
        gb, cb = kk.to(DEV, key_dtype).contiguous(), kk.clone()
        g.clock.add_(1)
        c.clock.add_(1)
        for l in range(2):
            g.touch(gb[l:l + 1], 0, n)
            c.touch(cb[l:l + 1], 0, n)
        adm[1].zero_()
        for l in range(2):
            g.insert(gb[l:l + 1], 0, n, adm=adm)
            c.insert(cb[l:l + 1], 0, n)
        g.reinit(adm, 2 * n, w32, s0, s1, 0, ev, ev, 0.25, 0.05, key)
        g.reinit(adm, 2 * n, wbf, r0, None, 0, ev, 1, 0.5, 0.05, key)
        assert by_key(g) == by_key(c)
        assert torch.equal(g.stats.cpu(), c.stats)
        # rows written in place: every present key reads its own way
        rows = gb.long()
        ok = rows >= 0
        assert torch.equal(g.keys[rows[ok]].cpu(), kk[ok.cpu()].long())
        na = int(adm[1])
        total_adm += na
        ways = adm[0][:na]
        ref = E.evict_init_rows(key, g.keys[ways], 0, ev, 0.05)
        assert torch.equal(w32[ways].cpu(), ref)
        assert torch.equal(wbf[ways].cpu(), ref.to(torch.bfloat16))
        assert bool((s0[ways] == 0.25).all()) and bool((s1[ways] == 0).all()) and bool((r0[ways] == 0.5).all())
    st = c.stats.tolist()
    assert st[1] > 0 and st[2] == 0 and total_adm == st[0]


def test_adversarial_set_admits_exactly_the_room():
    """more than 32 new keys of one set in one step: exactly the free room is admitted, the rest read zero and
    get no row; no key of the running step is evicted"""
    from hugectr_b200.embedding.collection import EmbeddingCollection, EmbeddingCollectionConfig, EmbeddingTableConfig
    cap, b = 64, 50
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(EmbeddingTableConfig("t", -1, 8, max_capacity=cap, evict_strategy="lru"), "k", "emb", "sum")
    e = EmbeddingCollection(cfg, b, {"k": 1}, DEV, torch.float32, Comm.single(DEV), CreateOptimizer(Optimizer_t.SGD),
                            key_dtype=torch.int64)
    ks = keys_of_set(0, cap // 32, 60, start=10**9)
    old, new = ks[:10], ks[10:50]
    lr, st = torch.tensor([0.1], device=DEV), torch.tensor([1], dtype=torch.int32, device=DEV)

    def step(keys):
        e.set_keys(torch.tensor(keys, dtype=torch.int64, device=DEV))
        e.forward(True)
        out = e.top_data["emb"].clone()
        e.top_grad["emb"].fill_(1.0)
        e.backward(lr, st)
        return out.view(b, -1)
    step((old * 5)[:b])
    ht = e._dyn_tables[("t", 0, 0)]
    before = {int(k): w for k, w in zip(*e.dump_table_local("t")[0][:2])}
    out = step(old + new)
    live = set(ht.dump()[0].tolist())
    assert set(old) <= live and len(live) == 32
    admitted = [k for k in new if k in live]
    assert len(admitted) == 22 and e.eviction_stats()[("t", 0)]["dropped"] == 18
    zero = (out.abs().sum(1) == 0).cpu()
    assert int(zero.sum()) == 18 and all(bool(zero[10 + i]) == (k not in live) for i, k in enumerate(new))
    after = {int(k): w for k, w in zip(*e.dump_table_local("t")[0][:2])}
    for k in old:        # trained: SGD with gradient 1 per occurrence
        assert torch.allclose(after[k], before[k] - 0.1, atol=1e-6)


@pytest.mark.parametrize("arm", ["adagrad", "rowwise_adagrad", "bf16"])
def test_training_matches_the_cpu_path(arm):
    """20 steps of a collection with one evicting table (two lookups, row-sharded over one rank), gradients
    that depend on the outputs: the live keys match the CPU path exactly after every step, the weights and
    state of the live keys within the tolerances of the fused-update tests"""
    opt = CreateOptimizer(Optimizer_t.RowWiseAdaGrad if arm == "rowwise_adagrad" else Optimizer_t.AdaGrad,
                          initial_accu_value=0.1, epsilon=1e-7)
    wdt = "bf16" if arm == "bf16" else "fp32"
    b, H, cap = 64, 2, 512
    batches = power_law_batches(20, 1, 2 * b * H, 4000, seed=9)
    eg, lg = _train_collection(Comm.single(DEV), "lfu", batches, cap, b, H, opt=opt, wdtype=wdt)
    ec, lc = _train_collection(Comm.single(CPU), "lfu", batches, cap, b, H, opt=opt, wdtype=wdt)
    assert lg == lc
    assert eg.eviction_stats()[("t", 0)]["evicted"] > 0
    (kg, wg, _, sg, _), = eg.dump_table_local("t")
    (kc, wc, _, sc, _), = ec.dump_table_local("t")
    assert torch.equal(kg, kc)
    # bf16: the stochastic rounding is keyed by arena position, and ways may differ between the paths
    tol = dict(rtol=2e-2, atol=2e-3) if wdt == "bf16" else dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(wg, wc, **tol)
    torch.testing.assert_close(sg[0], sc[0], **(dict(rtol=1e-2, atol=1e-3) if wdt == "bf16" else tol))


def test_model_fit_captures_the_step_graph_once(monkeypatch):
    """Model.fit with CUDA graphs and an evicting table: evictions happen, the step graph is captured once"""
    import torch.cuda as tc
    made = []

    class Counting(tc.CUDAGraph):
        def __init__(self, *a, **k):
            made.append(1)
            super().__init__(*a, **k)
    monkeypatch.setattr(tc, "CUDAGraph", Counting)
    m = _fit_model("lfu", device=DEV)
    m.fit(max_iter=60, display=5, eval_interval=0, snapshot=10**9)
    st = m.ebcs_train[0].eviction_stats()[("t", 0)]
    assert st["evicted"] > 0 and st["live"] == 64
    assert m._graph is not None and len(made) == 1


@pytest.mark.parametrize("strategy", ["lru", "lfu"])
def test_emulated_ranks_peer_memory_path_matches_the_oracle(strategy):
    from hugectr_b200.parallel.emu import run_ranks
    world, b, H, cap = 4, 32, 2, 512
    batches = power_law_batches(12, world, 2 * b * H, 20000, seed=4)

    def run(comm):
        e, lives = _train_collection(comm, strategy, batches, cap, b, H)
        assert e.fused
        return lives
    res = run_ranks(world, run, device=DEV)
    ref = oracle_lives(batches, world, strategy, cap, b, H)
    for step in range(len(batches)):
        for s in range(world):
            assert res[s][step] == ref[step][s], (step, s)


def test_checkpoint_round_trip_and_overfull_load():
    b, H, cap = 64, 2, 256
    batches = power_law_batches(10, 1, 2 * b * H, 3000, seed=2)
    e, lives = _train_collection(Comm.single(DEV), "lru", batches, cap, b, H)
    (k, w, _, sts, _), = e.dump_table_local("t")
    assert k.tolist() == lives[-1] and len(k) == cap
    e2, _ = _train_collection(Comm.single(DEV), "lru", [], cap, b, H, seed=99)
    e2.load_table_rows("t", k, w, sts)
    (k2, w2, _, sts2, _), = e2.dump_table_local("t")
    assert torch.equal(k2, k) and torch.equal(w2, w) and torch.equal(sts2[0], sts[0])
    e3, _ = _train_collection(Comm.single(DEV), "lru", [], cap, b, H)
    many = torch.tensor(keys_of_set(3, cap // 32, 40, start=10**6))
    with pytest.raises(RuntimeError, match=r"table t: shard 0 .*8 of 40"):
        e3.load_table_rows("t", many, torch.zeros(40, 8))
