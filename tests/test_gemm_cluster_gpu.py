"""The 2-CTA cluster GEMM (block_n 1000 + BN: each CTA loads half of the B tile and multicasts it, and a stage is
refilled only after the consumers of both CTAs released it) computes the same bits as the single-CTA kernel.
The K order of the accumulation does not depend on the tile, so any stage overwritten too early shows up as a
mismatch.  Shapes: long K (many passes over every stage), the DCNv2 cross shape, and ragged M / N / K."""
import pytest
import torch

from hugectr_b200.ops import gemm as G

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)


@pytest.mark.parametrize("b_mn", [True, False])
@pytest.mark.parametrize("M,N,K", [(6912, 512, 3456), (6912, 3456, 512), (1000, 200, 136), (130, 328, 16)])
def test_cluster_matches_single_cta(b_mn, M, N, K):
    torch.manual_seed(0)
    a = _mk((M, K), 0.5)
    b = _mk((K, N) if b_mn else (N, K), 0.5)
    bias = torch.randn(N, device="cuda")
    x0, xl = _mk((M, N)), _mk((M, N))
    kw = dict(b_mn=b_mn, bias=bias, x0=x0, xl=xl, flags=G.EPI_CROSS)
    ref = G.gemm_reference(a, b, False, b_mn, bias=bias, x0=x0, xl=xl, flags=G.EPI_CROSS | G.EPI_OUT_F32)
    for bn in (128, 256):
        one = G.gemm_bf16(a, b, block_n=bn, **kw)
        assert (one.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-2, bn
        for _ in range(2):
            pair = G.gemm_bf16(a, b, block_n=1000 + bn, **kw)
            assert torch.equal(pair, one), 1000 + bn
