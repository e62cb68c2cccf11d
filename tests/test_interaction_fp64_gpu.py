"""The DLRM dot interaction (csrc/interaction.cu and its fallback) against fp64, at its shape and alignment edges.

out[s] = [ mlp[s] | strict lower triangle of X X^T | 0 ] with X = [mlp[s]; emb[s]] (n rows of width D).
* forward: the passthrough columns are bit-exact and the pad column is +0; the triangle is held to the bf16
  wgmma bound ``2^-8 |ref| + 2 (D + 1) 2^-24 sum_d |x_i x_j|`` (tests/test_dense_path_fp64_gpu.py).
* backward: dX = (G + G^T) X, plus dout[:, :D] for the mlp row, held to the same bound over its n + 1 terms.
  dmlp and demb are filled with a sentinel first: both are overwritten, not accumulated into.
* every buffer is the contiguous [:B] prefix of a [B + 4, ...] allocation whose last rows must stay untouched.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_dense_path_fp64_gpu as DP  # noqa: E402
from hugectr_b200.ops import interaction as I  # noqa: E402
from hugectr_b200.ops import interaction_native as N  # noqa: E402

pytestmark = pytest.mark.gpu
f64 = torch.float64
DEV = "cuda"
SENTINEL = -77.0          # exactly representable in bf16


def _prefix(shape, B, fill=None, seed=None, scale=1.0):
    """contiguous [:B] prefix of a bf16 [B + 4, *shape] buffer: random (seeded) with NaN rows past B, so that a
    read past the batch poisons the result, or filled"""
    if fill is None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        base = (torch.randn((B + 4, *shape), generator=g, device=DEV) * scale).bfloat16()
        base[B:] = float("nan")
    else:
        base = torch.full((B + 4, *shape), fill, dtype=torch.bfloat16, device=DEV)
    return base, base[:B]


def oracle(mlp, emb, dout):
    """fp64 forward, its magnitudes, and fp64 dmlp / demb with theirs"""
    B, D = mlp.shape
    n = emb.shape[1] + 1
    x = torch.cat([mlp.unsqueeze(1), emb], 1).to(f64)                 # [B, n, D]
    z, zmag = x @ x.transpose(1, 2), x.abs() @ x.abs().transpose(1, 2)
    li, lj = torch.tril_indices(n, n, -1, device=DEV)
    tri, trimag = z[:, li, lj], zmag[:, li, lj]
    g = torch.zeros(B, n, n, dtype=f64, device=DEV)
    g[:, li, lj] = dout[:, D:D + li.numel()].to(f64)
    gs = g + g.transpose(1, 2)
    dx, dxmag = gs @ x, gs.abs() @ x.abs()
    dx[:, 0] += dout[:, :D].to(f64)
    dxmag[:, 0] += dout[:, :D].to(f64).abs()
    return tri, trimag, dx, dxmag


def run_and_check(B, n, D, seed=0, expect_native=None):
    w = D + n * (n - 1) // 2 + 1
    mb, mlp = _prefix((D,), B, seed=seed, scale=0.5)
    eb, emb = _prefix((n - 1, D), B, seed=seed + 1, scale=0.5)
    ob, out = _prefix((w,), B, fill=SENTINEL)
    db, dout = _prefix((w,), B, seed=seed + 2, scale=0.1)
    gmb, dmlp = _prefix((D,), B, fill=SENTINEL)
    geb, demb = _prefix((n - 1, D), B, fill=SENTINEL)
    if expect_native is not None:
        assert N.available(mlp, emb, out) == expect_native
        assert N.available(mlp, emb, dout, dmlp, demb) == expect_native
    I.interaction_fwd(mlp, emb, out)
    I.interaction_bwd(mlp, emb, dout, dmlp, demb)
    tri, trimag, dx, dxmag = oracle(mlp, emb, dout)
    torch.cuda.synchronize()
    for base, what in ((ob, "out"), (gmb, "dmlp"), (geb, "demb")):
        assert bool((base[B:] == SENTINEL).all()), f"{what}: rows B.. written"
    assert torch.equal(out[:, :D], mlp), "passthrough"
    assert bool((out[:, -1].view(torch.int16) == 0).all()), "pad column is not +0"
    DP.assert_sum(out[:, D:w - 1], tri, trimag, D, DP.BF16_R, f"triangle B={B} n={n} D={D}")
    DP.assert_sum(dmlp, dx[:, 0], dxmag[:, 0], n + 1, DP.BF16_R, f"dmlp B={B} n={n} D={D}")
    DP.assert_sum(demb, dx[:, 1:], dxmag[:, 1:], n + 1, DP.BF16_R, f"demb B={B} n={n} D={D}")


NS = [1, 2, 3, 9, 16, 17, 27, 31, 32]
DS = [16, 32, 48, 64, 80, 112, 128]


@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("B", [1, 2, 3, 5, 1057])
def test_interaction_native(B, n, D):
    """1057 samples are 265 tiles, more than 2 CTAs on each SM take in one pass: CTAs loop.  n = 27 gives an
    output width divisible by 8 (the 16-byte passthrough), the others the scalar one."""
    run_and_check(B, n, D, seed=B * 1000 + n * 10 + D, expect_native=True)


@pytest.mark.parametrize("n,D", [(27, 128), (32, 128), (2, 16), (17, 48)])
def test_interaction_native_full_batch(n, D):
    run_and_check(6912, n, D, seed=n + D, expect_native=True)


@pytest.mark.parametrize("n,D", [(33, 128), (27, 136), (27, 144), (2, 8)])
def test_interaction_fallback(n, D, monkeypatch):
    """shapes the kernels do not take run the fp32 fallback, under the same bound (fp32 matmuls: a model built
    earlier in the process may have allowed TF32)"""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    run_and_check(37, n, D, seed=n + D, expect_native=False)


def test_dispatch_rejects():
    """predicates only: nothing is launched on these tensors"""
    B, n, D = 8, 5, 64
    w = D + n * (n - 1) // 2 + 1
    bf = dict(dtype=torch.bfloat16, device=DEV)
    mlp, emb, out = torch.zeros(B, D, **bf), torch.zeros(B, n - 1, D, **bf), torch.zeros(B, w, **bf)
    dmlp, demb = torch.zeros_like(mlp), torch.zeros_like(emb)
    assert N.available(mlp, emb, out) and N.available(mlp, emb, out, dmlp, demb)
    shifted = lambda t: torch.zeros(t.numel() + 8, **bf)[1:1 + t.numel()].view(t.shape)  # noqa: E731
    for i in range(3):                                     # a base that is not 16-byte aligned
        ts = [mlp, emb, out]
        ts[i] = shifted(ts[i])
        assert ts[i].is_contiguous() and not N.available(*ts)
    assert not N.available(mlp, emb, out, shifted(dmlp), demb)
    assert not N.available(mlp, emb, out, dmlp, shifted(demb))
    assert not N.available(mlp, emb, out, torch.zeros(D, B, **bf).t(), demb)          # non-contiguous
    assert not N.available(mlp, emb, out, dmlp, torch.zeros(B, D, n - 1, **bf).transpose(1, 2))
    assert not N.available(mlp, emb, out, dmlp.float(), demb)                          # non-bf16
    assert not N.available(mlp, emb, out, dmlp, demb.float())


def test_interaction_layer_bench_shape():
    """InteractionLayer at the bench's --model dlrm shape, forward and backward, twice with different inputs"""
    from hugectr_b200.enums import Layer_t
    from hugectr_b200.layers import LAYER_REGISTRY, BuildCtx, ParamArena, TensorBag
    from hugectr_b200.solver import CreateSolver, DenseLayer
    B, n, D = 6912, 27, 128
    dev = torch.device(DEV)
    ctx = BuildCtx(ParamArena(), dev, torch.bfloat16, B, True, CreateSolver(), True)
    xs = []
    for name, shape in (("mlp", (B, D)), ("emb", (B, n - 1, D))):
        t = TensorBag(name, shape, torch.bfloat16)
        t.data = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        t.grad = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        xs.append(t)
    layer = LAYER_REGISTRY[Layer_t.Interaction](DenseLayer(Layer_t.Interaction, ["mlp", "emb"], ["out"]), xs, ctx)
    layer.allocate()
    o = layer.outputs[0]
    for seed in (10, 20):
        g = torch.Generator(device=DEV).manual_seed(seed)
        for t in xs:
            t.data.copy_(torch.randn(t.data.shape, generator=g, device=DEV) * 0.5)
            t.grad.fill_(SENTINEL)
        o.grad.copy_(torch.randn(o.grad.shape, generator=g, device=DEV) * 0.1)
        layer.fprop(True)
        layer.bprop()
        tri, trimag, dx, dxmag = oracle(xs[0].data, xs[1].data, o.grad)
        torch.cuda.synchronize()
        assert torch.equal(o.data[:, :D], xs[0].data)
        assert bool((o.data[:, -1].view(torch.int16) == 0).all())
        DP.assert_sum(o.data[:, D:-1], tri, trimag, D, DP.BF16_R, "layer triangle")
        DP.assert_sum(xs[0].grad, dx[:, 0], dxmag[:, 0], n + 1, DP.BF16_R, "layer dmlp")
        DP.assert_sum(xs[1].grad, dx[:, 1:], dxmag[:, 1:], n + 1, DP.BF16_R, "layer demb")
