"""Delta export on the H100: the stamp kernel against the CPU path (random lists, an overflowed counter, an empty
list, rows at the slice ends), the kernel inside a replayed CUDA graph reading the clock on the device, the exact
delta of a graph-captured model, tracking that leaves a graph-captured model's training bit-identical, and the
serving round trip with fp8_quant off and on."""
from types import SimpleNamespace

import pytest
import torch

from hugectr_b200.embedding import ops as E

from test_embedding_delta_cpu import (EV, INPUTS, batches, build_model, check_exact_delta,
                                      check_serving_round_trip)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _lists(rows, seed):
    """(unique rows int64 [max_unique], counter) cases: random, overflowed, empty, the slice ends"""
    g = torch.Generator().manual_seed(seed)
    mu = 1000
    perm = torch.randperm(rows, generator=g)[:mu]
    ends = torch.tensor([0, rows - 1, rows // 2, 1, rows - 2])
    return [(perm, 700), (perm, mu + 37), (perm, 0), (torch.cat([ends, perm[:mu - 5]]), 5),
            (torch.cat([ends, perm[:mu - 5]]), mu)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_stamp_kernel_matches_cpu_path(seed):
    rows = 5000
    for i, (lst, cnt) in enumerate(_lists(rows, seed)):
        start = torch.randint(0, 50, (rows,), dtype=torch.int32, generator=torch.Generator().manual_seed(i))
        clock = torch.tensor([1000 + i], dtype=torch.int64)
        dev_st = start.to(DEV)
        ws = SimpleNamespace(rows=lst.to(DEV), counter=torch.tensor([cnt], dtype=torch.int32, device=DEV),
                             max_unique=lst.numel())
        E.stamp_rows(dev_st, ws, clock.to(DEV))
        cpu_st = start.clone()
        E.stamp_rows(cpu_st, SimpleNamespace(ref_rows=lst[:min(cnt, lst.numel())]), clock)
        assert torch.equal(dev_st.cpu(), cpu_st), (seed, i)


def test_stamp_kernel_reads_the_clock_on_the_device_in_a_graph():
    rows, K = 4096, 6
    stamp = torch.zeros(rows, dtype=torch.int32, device=DEV)
    clock = torch.zeros(1, dtype=torch.int64, device=DEV)
    lst = torch.zeros(512, dtype=torch.int64, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = SimpleNamespace(rows=lst, counter=cnt, max_unique=lst.numel())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.stamp_rows(stamp, ws, clock)             # (warm-up outside the capture)
    torch.cuda.current_stream().wait_stream(s)
    stamp.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        clock.add_(1)
        E.stamp_rows(stamp, ws, clock)
    want = torch.zeros(rows, dtype=torch.int32)
    gen = torch.Generator().manual_seed(5)
    for step in range(1, K + 1):
        n = int(torch.randint(0, 512, (1,), generator=gen))
        rs = torch.randperm(rows, generator=gen)[:512]
        lst.copy_(rs)
        cnt.fill_(n)
        g.replay()
        want[rs[:n]] = step
    torch.cuda.synchronize()
    assert int(clock) == K
    assert torch.equal(stamp.cpu(), want)


def test_exact_delta_gpu(tmp_path):
    check_exact_delta(DEV, str(tmp_path), graph=True)


def _preload_dynamic(m, bs):
    """every key of the dynamic table that the batches hold, with fixed values: a new key's initial row is the one a
    concurrent insert hands out, so only preloaded keys start from the same values in two runs"""
    keys = torch.tensor(sorted({int(k) for _, per in bs for k in per["c"].reshape(-1) if k >= 0}))
    vals = torch.randn(keys.numel(), EV, generator=torch.Generator().manual_seed(2)) * 0.05
    m.ebcs_train[0].load_table_rows("tc", keys, vals)


def test_tracking_does_not_perturb_training():
    """the same model with and without tracking, trained through the captured step: the loss of every step, the
    dense weights and optimizer state, and every table's rows and optimizer state by key are bit-identical.  Every key
    occurs at most once per table and step: the sparse update sums a row's repeated occurrences in an order that can
    vary between runs (in the last bit), tracked or not."""
    bs = batches(10, seed=6, distinct=True)
    res = []
    for track in (True, False):
        m = build_model(DEV, track=track, graph=True)
        _preload_dynamic(m, bs)
        losses = []
        for hb, _ in bs:
            m.train_on_host_batch(hb)
            losses.append(m.get_current_loss())
        torch.cuda.synchronize()
        assert m._graph is not None                    # the later steps replayed the captured step
        e = m.ebcs_train[0]
        assert all((g.stamp is not None) == track for g in e.groups)
        dense = [None if x is None else x.clone() for x in (m.arena.weights, m.opt_s0, m.opt_s1)]
        res.append((losses, dense, {t: e.dump_table_local(t) for _, _, t, _ in INPUTS}, int(e.evict_clock)))
    (l1, d1, t1, c1), (l2, d2, t2, c2) = res
    assert l1 == l2 and c1 == c2 == len(bs)
    for x, y in zip(d1, d2):
        assert (x is None and y is None) or torch.equal(x, y)
    for t in t1:
        for (k1, w1, _, s1, _), (k2, w2, _, s2, _) in zip(t1[t], t2[t]):
            assert torch.equal(k1, k2) and torch.equal(w1, w2), t
            for x, y in zip(s1, s2):
                assert (x is None and y is None) or torch.equal(x, y), t


def test_serving_round_trip_gpu(tmp_path):
    check_serving_round_trip(DEV, str(tmp_path), graph=True)
