"""Block-scaled fp8 (MX) GEMM: quantiser against the PyTorch reference (bit exact), tensor-core GEMM
(fp8 wgmma per 32-wide scale slice, scaled promotion) against the fp32 product of the de-quantised operands."""
import pytest
import torch

from hugectr_b200.ops import gemm as G
from hugectr_b200.ops import mxfp8 as MX


def test_mx_quantize_reference_roundtrip_cpu():
    torch.manual_seed(0)
    x = torch.randn(200, 256) * torch.logspace(-3, 2, 256).unsqueeze(0)
    q, sf = MX.mx_quantize_reference(x)
    xd = MX.mx_dequantize(q, sf, 200, 256)
    rel = (xd - x).abs() / x.abs().clamp(min=1e-6)
    assert rel.median() < 0.04                                # e4m3: 3 mantissa bits
    blk = (xd - x).view(200, 8, 32).abs().amax(-1) / x.view(200, 8, 32).abs().amax(-1)
    assert blk.max() < 0.07                                  # error relative to the block's largest element
    y = MX.gemm_mxfp8(q, sf, q, sf, 200, 200, 256, flags=G.EPI_OUT_F32)
    assert torch.allclose(y, xd @ xd.t(), rtol=1e-5, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("transposed", [False, True])
def test_mx_quantize_kernel_matches_reference(transposed):
    torch.manual_seed(1)
    x = (torch.randn(300, 384) * torch.logspace(-2, 1, 384).unsqueeze(0)).to(torch.bfloat16)
    xin = x.t().contiguous().cuda() if transposed else x.cuda()
    q, sf = MX.mx_quantize(xin, transposed=transposed)
    qr, sfr = MX.mx_quantize_reference(x)
    assert torch.equal(sf.cpu(), sfr)              # same scale rule on both sides
    assert torch.equal(q.cpu(), qr)                # and the same round-to-nearest-even of the scaled values
    xd = MX.mx_dequantize(q, sf, 300, 384)
    blk = (xd - x.float()).view(300, 12, 32).abs().amax(-1) / x.float().view(300, 12, 32).abs().amax(-1).clamp(min=1e-20)
    assert blk.max() < 0.07


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(128, 128, 128), (256, 384, 512), (6912, 1024, 3456), (300, 200, 640)])
def test_gemm_mxfp8_matches_dequantised_product(shape):
    M, N, K = shape
    torch.manual_seed(2)
    a = (torch.randn(M, K) * 0.5).to(torch.bfloat16).cuda()
    b = (torch.randn(N, K) * 0.1).to(torch.bfloat16).cuda()
    bias = torch.randn(N).cuda()
    aq, sfa = MX.mx_quantize(a)
    bq, sfb = MX.mx_quantize(b)
    out = MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, bias=bias, flags=G.EPI_RELU)
    ref = torch.relu(MX.mx_dequantize(aq, sfa, M, K).cuda() @ MX.mx_dequantize(bq, sfb, N, K).cuda().t() + bias)
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err < 2e-2 * max(scale, 1.0), (err, scale)       # bf16 output rounding only
    full = torch.relu(a.float() @ b.float().t() + bias)
    rel = (out.float() - full).norm() / full.norm()
    assert rel < 0.06, rel                                   # quantisation error of the MX format


@pytest.mark.gpu
def test_mlp_layer_fp8_forward_close_to_bf16():
    """Solver.use_fp8_mlp: the MLP forward runs on the MX fp8 GEMM and stays within the format's error of the
    bf16 layer; backward (bf16) is unchanged"""
    import hugectr_b200 as hugectr
    from hugectr_b200.layers import LAYER_REGISTRY, BuildCtx, ParamArena, TensorBag
    from hugectr_b200.solver import CreateSolver, DenseLayer
    outs = {}
    for fp8 in (False, True):
        arena = ParamArena()
        solver = CreateSolver(use_mixed_precision=True, use_fp8_mlp=fp8)
        ctx = BuildCtx(arena, torch.device("cuda"), torch.bfloat16, 512, True, solver, True)
        x = TensorBag("x", (512, 256), torch.bfloat16)
        g = torch.Generator().manual_seed(5)
        x.data = (torch.randn(512, 256, generator=g) * 0.5).to(torch.bfloat16).cuda()
        x.grad = torch.zeros(512, 256, dtype=torch.bfloat16, device="cuda")
        cfg = DenseLayer(hugectr.Layer_t.MLP, ["x"], ["y"], num_outputs=[384, 128, 1],
                         activations=[hugectr.Activation_t.Relu, hugectr.Activation_t.Relu, hugectr.Activation_t.Non])
        layer = LAYER_REGISTRY[hugectr.Layer_t.MLP](cfg, [x], ctx)
        arena.finalize(torch.device("cuda"), True)
        layer.allocate()
        arena.init_params(3)
        layer.fprop(True)
        assert bool(getattr(layer, "_fp8_bufs", None)) == fp8
        layer.outputs[0].grad.fill_(0.01)
        layer.bprop()
        outs[fp8] = (layer.outputs[0].data.float().clone(), x.grad.float().clone())
    y0, y1 = outs[False][0], outs[True][0]
    assert (y0 - y1).norm() / y0.norm() < 0.08
    # (bf16 backward through ReLU masks taken from the fp8 forward: a few mask flips per row)
    assert (outs[False][1] - outs[True][1]).norm() / outs[False][1].norm() < 0.4
