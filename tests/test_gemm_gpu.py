"""wgmma GEMM vs fp32 PyTorch oracle (reference test pattern: test/utest/core23_layer_test/mlp_test.cpp)."""
import pytest
import torch

from hugectr_b200.ops import gemm as G

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(256, 128, 64), (6912, 1024, 512), (1000, 200, 136), (128, 512, 3456)])
def test_gemm_majors(a_mn, b_mn, M, N, K):
    torch.manual_seed(0)
    a = _mk((K, M) if a_mn else (M, K), 0.5)
    b = _mk((K, N) if b_mn else (N, K), 0.5)
    out = G.gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn)
    ref = G.gemm_reference(a, b, a_mn, b_mn, flags=G.EPI_OUT_F32)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 1e-2, err


@pytest.mark.parametrize("bn", [0, 64, 128, 256, 1064, 1128, 1256])
def test_gemm_bias_relu(bn):
    torch.manual_seed(1)
    M, N, K = 1024, 512, 256
    a, b = _mk((M, K)), _mk((K, N), 0.1)
    bias = torch.randn(N, device="cuda")
    out = G.gemm_bf16(a, b, b_mn=True, bias=bias, flags=G.EPI_RELU, block_n=bn)
    ref = G.gemm_reference(a, b, False, True, bias=bias, flags=G.EPI_RELU | G.EPI_OUT_F32)
    assert (out.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-2


def test_gemm_mask_dgrad():
    torch.manual_seed(2)
    M, N, K = 2048, 384, 512
    dy, w = _mk((M, K)), _mk((N, K), 0.1)
    act = torch.relu(_mk((M, N)))
    out = G.gemm_bf16(dy, w, mask=act, flags=G.EPI_MASK)
    ref = G.gemm_reference(dy, w, mask=act, flags=G.EPI_MASK | G.EPI_OUT_F32)
    assert (out.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-2


@pytest.mark.parametrize("splits", [1, 4])
def test_gemm_wgrad_splitk(splits):
    torch.manual_seed(3)
    Kb, M, N = 6912, 512, 256
    x, dy = _mk((Kb, M)), _mk((Kb, N), 0.1)
    out = torch.zeros(M, N, device="cuda")
    G.gemm_bf16(x, dy, out, a_mn=True, b_mn=True, flags=G.EPI_ATOMIC, splits=splits)
    ref = x.float().t() @ dy.float()
    assert (out - ref).abs().max().item() <= 1e-2 * ref.abs().max().item() + 1e-2


def test_gemm_cross_epilogue():
    torch.manual_seed(4)
    M, N, K = 1024, 3456, 512
    h, v = _mk((M, K), 0.2), _mk((K, N), 0.1)
    x0, xl = _mk((M, N)), _mk((M, N))
    bias = torch.randn(N, device="cuda")
    aux = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    out = G.gemm_bf16(h, v, b_mn=True, bias=bias, x0=x0, xl=xl, aux=aux, flags=G.EPI_CROSS)
    aux_ref = torch.empty(M, N, device="cuda")
    ref = G.gemm_reference(h, v, False, True, bias=bias, x0=x0, xl=xl, aux=aux_ref,
                           flags=G.EPI_CROSS | G.EPI_OUT_F32)
    assert (aux.float() - aux_ref).abs().max().item() <= 2e-2 * aux_ref.abs().max().item() + 1e-2
    assert (out.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 2e-2


@pytest.mark.parametrize("bn", [1064, 1128, 1256])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(6912, 1024, 512), (1000, 328, 136), (384, 512, 3456), (130, 72, 200)])
def test_gemm_cluster_multicast(bn, a_mn, b_mn, M, N, K):
    """2-CTA clusters sharing the B tile by TMA multicast, incl. an odd number of M tiles (the second CTA of the
    last cluster is past M) and the 64-wide tile whose one B chunk the first CTA multicasts"""
    torch.manual_seed(0)
    a = _mk((K, M) if a_mn else (M, K), 0.5)
    b = _mk((K, N) if b_mn else (N, K), 0.5)
    out = G.gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, block_n=bn)
    ref = G.gemm_reference(a, b, a_mn, b_mn, flags=G.EPI_OUT_F32)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 1e-2, err


@pytest.mark.parametrize("bn", [0, 128, 1064, 1128, 1256])
@pytest.mark.parametrize("M,N,K,masked", [(6912, 512, 1024, True), (300, 200, 136, True), (1000, 328, 512, False)])
def test_gemm_fused_bias_gradient(bn, M, N, K, masked):
    """colsum= accumulates the column sums of the (bf16) output (a reduction after the GEMM, on every tile
    configuration); ragged M / N edges must not contribute"""
    torch.manual_seed(7)
    dy, w = _mk((M, K), 0.5), _mk((N, K), 0.5)
    mask = (torch.randn(M, N, device="cuda") > 0).to(torch.bfloat16) if masked else None
    cs = torch.full((N,), 1.5, device="cuda")
    out = G.gemm_bf16(dy, w, mask=mask, flags=G.EPI_MASK if masked else 0, block_n=bn, colsum=cs)
    torch.cuda.synchronize()
    ref = out.float().sum(0) + 1.5
    assert (cs - ref).abs().max().item() <= 1e-3 * ref.abs().max().item() + 1e-2


def test_gemm_rejects_unknown_cluster_codes():
    a, b = _mk((256, 64)), _mk((128, 64))
    with pytest.raises(RuntimeError, match="rc=-11"):
        G.gemm_bf16(a, b, block_n=2128)
