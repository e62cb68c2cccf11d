"""The element-wise optimizer rules (csrc/optim.cuh, ops/optim.py) and the optimizer state they start from.

GPU: the dense optimizer (dense_opt_kernel) against the host rule for each of the seven rules, on n = 4k + 3
weights (the float4 body and the scalar tail), with the bf16 weight copy, gradient zeroing and a loss scaler.
Error bound: the kernels are built with --use_fast_math, so square roots and divisions are approximate
(a few fp32 ulp each) and products may be fused.  Every rule is old + update with O(1) operands here, so
the device and the fp32 host values agree within 1e-5 relative plus 1e-6 absolute.  FTRL is the exception:
z_new = z + g + (sqrt(n + beta) - sqrt(n_new + beta)) w / lr cancels, so its rounding is relative to the
terms, not to the result (TOL_U units of fp32 rounding of their magnitudes); w_new = (+-lambda1 - z_new) / q
carries that error divided by q.

CPU: how many per-weight state arrays each optimizer gets, and their initial values, wherever optimizer
state is allocated: the dense model optimizer, an embedding-collection model-parallel group, a legacy
SparseEmbedding and a CreateETC (host parameter server) table.
"""
import types

import pytest
import torch

import hugectr_b200 as hugectr
from hugectr_b200.enums import Optimizer_t as O
from hugectr_b200.ops import dense as D
from hugectr_b200.ops.optim import opt_reference

U = 2.0 ** -24
TOL_U = 32
ELEMENTWISE = [O.SGD, O.AdaGrad, O.Adam, O.Ftrl, O.MomentumSGD, O.Nesterov, O.RMSProp]
STATES = {O.SGD: 0, O.AdaGrad: 1, O.Adam: 2, O.Ftrl: 2, O.MomentumSGD: 1, O.Nesterov: 1, O.RMSProp: 1,
          O.RowWiseAdaGrad: 0}
HP = dict(scaler=1024.0, beta1=0.875, beta2=0.9375, epsilon=1e-7, lambda1=0.05, lambda2=0.1, ftrl_beta=1.0,
          momentum=0.9)
LR = 0.01


def _inputs(opt, n, gen):
    w = torch.randn(n, generator=gen)
    g = torch.randn(n, generator=gen) * HP["scaler"]
    positive = opt in (O.AdaGrad, O.RMSProp)
    s0 = torch.rand(n, generator=gen) + 0.1 if positive else torch.randn(n, generator=gen) * 0.1
    s1 = torch.rand(n, generator=gen)
    ns = STATES[opt]
    return w, g, s0 if ns >= 1 else None, s1 if ns >= 2 else None


@pytest.mark.gpu
@pytest.mark.parametrize("opt,step", [(o, 1) for o in ELEMENTWISE] + [(O.Adam, 7)])
def test_dense_optimizer_kernel_matches_host_rule(opt, step):
    n = 4 * 1000 + 3
    w, g, s0, s1 = _inputs(opt, n, torch.Generator().manual_seed(int(opt.value) * 10 + step))
    dev = torch.device("cuda")
    cu = [None if x is None else x.to(dev) for x in (w, g, s0, s1)]
    w16 = torch.zeros(n, dtype=torch.bfloat16, device=dev)
    D.dense_opt_step(opt, cu[0], cu[1], w16, cu[2], cu[3], torch.full((1,), LR, device=dev),
                     torch.full((1,), step, dtype=torch.int32, device=dev), HP, zero_grad=True)
    torch.cuda.synchronize()
    ref = [None if x is None else x.clone() for x in (w, s0, s1)]
    opt_reference(opt, ref[0], ref[1], ref[2], g, HP, LR, step)
    got = [None if x is None else x.cpu() for x in (cu[0], cu[2], cu[3])]
    assert torch.equal(cu[1].cpu(), torch.zeros(n)), "the gradient is zeroed"
    assert torch.equal(w16.cpu(), got[0].to(torch.bfloat16)), "w16 is the weights rounded to nearest"
    if opt == O.Ftrl:
        fb, gg = HP["ftrl_beta"], g / HP["scaler"]
        mag = s0.abs() + gg.abs() + ((s1 + fb).sqrt() + (s1 + gg * gg + fb).sqrt()) * w.abs() / LR
        tol_z = TOL_U * U * mag
        q = (ref[2] + fb).sqrt() / LR + HP["lambda2"]
        assert ((got[1] - ref[1]).abs() <= tol_z).all()
        torch.testing.assert_close(got[2], ref[2], rtol=1e-5, atol=1e-6)
        assert ((got[0] - ref[0]).abs() <= tol_z / q + 1e-6 + 1e-5 * ref[0].abs()).all()
        return
    for a, b in zip(got, ref):
        if b is not None:
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def _opts():
    for t in STATES:
        if t == O.Adam:
            yield t, hugectr.Update_t.LazyGlobal      # num_states counts a third array that is never allocated
        yield t, hugectr.Update_t.Global


def _check(s0, s1, t, accu):
    ns = STATES[t]
    assert (s0 is not None, s1 is not None) == (ns >= 1, ns >= 2)
    if s0 is not None:
        assert torch.equal(s0, torch.full_like(s0, accu if t == O.AdaGrad else 0.0))
    if s1 is not None:
        assert torch.equal(s1, torch.zeros_like(s1))


@pytest.mark.parametrize("t,upd", list(_opts()))
def test_optimizer_state_layout_and_initial_values(t, upd):
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.embedding.offloaded import CachedSparseEmbeddingRuntime
    from hugectr_b200.embedding.sparse_embedding import SparseEmbeddingRuntime
    from hugectr_b200.model import Model
    from hugectr_b200.parallel.comm import Comm
    accu = 0.25
    opt = hugectr.CreateOptimizer(t, upd, initial_accu_value=accu)
    dev = torch.device("cpu")
    # embedding-collection model-parallel group (row-wise AdaGrad: one fp32 accumulator per row)
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup([EmbeddingTableConfig("0", 50, 4, opt_params=opt)], ["d0"], "emb", ["sum"])
    e = EmbeddingCollection(cfg, 3, {"d0": 2}, dev, torch.float32, Comm.single(dev),
                            hugectr.CreateOptimizer(O.SGD))
    (grp,) = e.groups
    assert grp.kind == "mp"
    if t == O.RowWiseAdaGrad:
        assert grp.s0.shape == (grp.rows,) and grp.s1 is None
        assert torch.equal(grp.s0, torch.full_like(grp.s0, accu))
        return
    _check(grp.s0, grp.s1, t, accu)
    # dense model optimizer
    m = types.SimpleNamespace(opt_params=opt, device=dev, arena=types.SimpleNamespace(weights=torch.zeros(10)),
                              solver=types.SimpleNamespace(lr=0.1, scaler=1.0), mixed=False)
    Model._create_dense_optimizer(m)
    _check(m.opt_s0, m.opt_s1, t, accu)
    # legacy SparseEmbedding, in memory and behind the host parameter server (CreateETC)
    se = hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 0, 4, "sum", "emb",
                                 "data", slot_size_array=[20, 20], optimizer=opt)
    se.max_vocabulary_size_per_gpu = 16
    prm = hugectr.DataReaderSparseParam("data", 1, True, 2)
    rt = SparseEmbeddingRuntime(se, prm, None, 4, dev, torch.float32, Comm.single(dev), opt, torch.int64)
    _check(rt.s0, rt.s1, t, accu)
    etc = CachedSparseEmbeddingRuntime(se, prm, None, 4, dev, torch.float32, Comm.single(dev), opt, torch.int64,
                                       ps_type=hugectr.TrainPSType_t.Cached)
    assert etc.nstates == len(etc.ps.s) == len(etc.state_cache) == STATES[t]
    _check(*(etc.ps.s + [None, None])[:2], t, accu)
