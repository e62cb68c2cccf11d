"""Weighted embedding-collection lookups on the H100: the lookup and every update path against the CPU path
(which test_embedding_weighted_cpu.py holds to the fp64 oracle), the all-ones invariant bit for bit, emulated
ranks on the peer-memory path and one CUDA-graph capture for a weighted Model.fit."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_embedding_weighted_cpu import (CPU, HOT, dump_full, flat, load_tables, make_batch,  # noqa: E402
                                         make_collection, make_tables, oracle_forward, step, _model)

from hugectr_b200.enums import Optimizer_t  # noqa: E402
from hugectr_b200.parallel.comm import Comm  # noqa: E402
from hugectr_b200.solver import CreateOptimizer  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None

OPTS = {"sgd": (Optimizer_t.SGD, {}), "adagrad": (Optimizer_t.AdaGrad, dict(initial_accu_value=0.1, epsilon=1e-7)),
        "adam": (Optimizer_t.Adam, {}), "rowwise": (Optimizer_t.RowWiseAdaGrad, dict(initial_accu_value=0.1))}
# path -> (ev, plan, power-law keys, batch): light / medium rows at uniform keys, heavy rows (> 64 occurrences) at
# power-law keys, the accumulate path at a width that is not a multiple of 4, and a data-parallel table
PATHS = {"indexed": (16, "table", False, 64), "heavy": (16, "table", True, 512), "accum": (6, "table", False, 64),
         "dp": (16, "dp", False, 64)}


def _opt(name):
    o, kw = OPTS[name]
    return CreateOptimizer(o, **kw)


def _tables(e, ev):
    return dump_full(e, (50, 7, 300), ev)


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("wdtype,sdtype", [("fp32", "fp32"), ("bf16", "fp32"), ("fp32", "bf16"), ("bf16", "bf16")])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_lookup_and_update_match_cpu(path, opt, wdtype, sdtype, combiner):
    if opt == "rowwise" and sdtype == "bf16":
        pytest.skip("row-wise AdaGrad keeps an fp32 accumulator")
    ev, plan, pl, B = PATHS[path]
    gen = torch.Generator().manual_seed(7)
    tables = make_tables(gen, ev=ev)
    sdt = torch.bfloat16 if sdtype == "bf16" else torch.float32
    kw = dict(plan=plan, combiner=combiner, opt=_opt(opt), ev=ev, weight_dtype=wdtype, state_dtype=sdt)
    eg = make_collection(DEV, Comm.single(DEV), B, HOT, **kw)
    ec = make_collection(CPU, Comm.single(CPU), B, HOT, **kw)
    load_tables(eg, tables); load_tables(ec, tables)
    if path in ("indexed", "heavy"):
        assert any(getattr(g, "indexed", False) for g in eg.groups)
    bf = wdtype == "bf16" or sdtype == "bf16"
    # the second lookup reads updated tables: fp32 sums in another order, amplified by Adam's normalisation
    tol = dict(rtol=2e-2, atol=2e-3) if bf else dict(rtol=1e-3, atol=1e-4)
    for it in range(2):
        keys, wts = make_batch(gen, B, HOT, power_law=pl)
        grad = torch.randn(B, 3 * ev, generator=gen) * 0.1
        og, oc = step(eg, keys, wts, grad), step(ec, keys, wts, grad)
        torch.cuda.synchronize()
        assert torch.isfinite(og).all()
        torch.testing.assert_close(og, oc, **(dict(rtol=1e-4, atol=1e-5) if it == 0 else tol))
    tg, tc = _tables(eg, ev), _tables(ec, ev)
    for n in tc:
        torch.testing.assert_close(tg[n], tc[n], **tol)


def test_forward_matches_fp64_oracle():
    gen = torch.Generator().manual_seed(3)
    tables = make_tables(gen)
    for combiner in ("sum", "mean"):
        e = make_collection(DEV, Comm.single(DEV), 128, HOT, combiner=combiner)
        load_tables(e, tables)
        keys, wts = make_batch(gen, 128, HOT)
        e.set_keys(flat(keys).int().to(DEV)); e.set_weights(flat(wts).to(DEV)); e.forward()
        out = e.top_data["emb"].double().cpu()
        assert (out - oracle_forward(tables, keys, wts, combiner)).abs().max().item() < 1e-5


@pytest.mark.parametrize("combiner", ["sum", "mean"])
@pytest.mark.parametrize("plan", ["table", "dp"])
def test_adagrad_step_matches_fp64_oracle_on_device(combiner, plan):
    from test_embedding_weighted_cpu import test_adagrad_step_matches_fp64_oracle
    test_adagrad_step_matches_fp64_oracle(combiner, plan, dev=DEV)


def _dyadic(gen, B, w):
    """gradients that are multiples of 2^-12: every fp32 sum of them is exact, so the counting sort's order of
    a row's entries cannot change a bit"""
    return torch.randint(-64, 65, (B, w), generator=gen).float() / 4096


def _ones_pair(dev, comm, B, ev=16, **kw):
    ew = make_collection(dev, comm, B, HOT, ev=ev, **kw)
    eu = make_collection(dev, comm, B, HOT, ev=ev, weighted=(), **kw)
    return ew, eu


def _ones_run(ew, eu, batches, ev, rows=None):
    for keys, wts, grad in batches:
        ow = step(ew, keys, wts, grad, rows=rows)
        ou = step(eu, keys, wts, grad, rows=rows, weights=False)
        assert torch.equal(ow, ou)
    torch.cuda.current_stream().synchronize()      # (emulated ranks: only this rank's stream)
    # by key: a dynamic table's key -> row map depends on the order its inserts land in
    for n in ("0", "1", "2"):
        for pw, pu in zip(ew.dump_table_local(n), eu.dump_table_local(n)):
            assert torch.equal(pw[0], pu[0]) and torch.equal(pw[1], pu[1])
            for a, b in zip(pw[3], pu[3]):
                assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.parametrize("path", list(PATHS) + ["evict", "grow"])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
@pytest.mark.parametrize("wdtype", ["fp32", "bf16"])
def test_all_ones_weights_reproduce_unweighted_bits(path, combiner, wdtype):
    ev, plan, pl, B = PATHS.get(path, (16, "table", True, 256))
    dyn = {"evict": "lru", "grow": "grow"}.get(path)
    if dyn and wdtype == "bf16":
        pytest.skip("bf16 stochastic rounding is keyed by arena row, which a dynamic table assigns in insert order")
    gen = torch.Generator().manual_seed(9)
    tables = make_tables(gen, ev=ev)
    ew, eu = _ones_pair(DEV, Comm.single(DEV), B, ev=ev, plan=plan, combiner=combiner, opt=_opt("adagrad"),
                        weight_dtype=wdtype, dynamic=dyn)
    load_tables(ew, tables); load_tables(eu, tables)       # (dynamic: the same row per key in both)
    batches = []
    for _ in range(3):
        keys, wts = make_batch(gen, B, HOT, power_law=pl, variable=False, ones=True)
        batches.append((keys, wts, _dyadic(gen, B, 3 * ev)))
    _ones_run(ew, eu, batches, ev)


@pytest.mark.parametrize("plan", ["row", "column", "dp"])
def test_emulated_ranks_peer_memory_path(plan):
    """fused (peer-memory) exchange on emulated ranks: weights travel with the keys; equal to one process, and
    all-ones weights reproduce the unweighted row-sharded bits (its bags take the requester-side split)"""
    from hugectr_b200.parallel.emu import run_ranks
    world, b = 4, 32
    gen = torch.Generator().manual_seed(13)
    tables = make_tables(gen)
    batches = [make_batch(gen, b * world, HOT) + (torch.randn(b * world, 48, generator=gen) * 0.1,) for _ in range(2)]
    ones = [make_batch(gen, b * world, HOT, variable=False, ones=True) + (_dyadic(gen, b * world, 48),)
            for _ in range(2)]
    one = make_collection(CPU, Comm.single(CPU), b * world, HOT, combiner="mean")
    load_tables(one, tables)
    ref = [step(one, k, w, g) for (k, w, g) in batches]
    ref_tab = dump_full(one, (50, 7, 300))

    def rank_fn(comm):
        rows = slice(comm.rank * b, (comm.rank + 1) * b)
        e = make_collection(comm.device, comm, b, HOT, plan=plan, combiner="mean")
        assert e.fused
        load_tables(e, tables)
        for (k, w, g), r in zip(batches, ref):
            out = step(e, k, w, g, rows=rows)
            torch.cuda.current_stream().synchronize()
            torch.testing.assert_close(out, r[rows], rtol=1e-4, atol=1e-5)
        comm.barrier()
        got = dump_full(e, (50, 7, 300))
        for n in ref_tab:
            if got[n] is not None:
                m = ~torch.isnan(got[n])
                torch.testing.assert_close(got[n][m], ref_tab[n][m], rtol=1e-4, atol=1e-5)
        ew, eu = _ones_pair(comm.device, comm, b, plan=plan, combiner="sum", opt=_opt("adagrad"))
        load_tables(ew, tables); load_tables(eu, tables)
        _ones_run(ew, eu, ones, 16, rows=rows)
        return True
    assert all(run_ranks(world, rank_fn, device=DEV))


def test_model_fit_captures_the_step_graph_once(monkeypatch, tmp_path):
    import torch.cuda as tc
    made = []

    class Counting(tc.CUDAGraph):
        def __init__(self, *a, **k):
            made.append(1)
            super().__init__(*a, **k)
    monkeypatch.setattr(tc, "CUDAGraph", Counting)
    m = _model(tmp_path, device=DEV)
    m.compile()
    assert m.ebcs_train[0].has_weights
    m.fit(max_iter=20, display=5, eval_interval=0, snapshot=10**9)
    assert m._graph is not None and len(made) == 1
    assert torch.isfinite(torch.tensor(m.get_current_loss()))
