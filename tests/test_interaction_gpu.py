"""wgmma dot-interaction vs the fp32 oracle (shapes of test/utest/core23_layer_test/interaction_layer_test.cpp:291-320)."""
import pytest
import torch

from hugectr_b200.ops import interaction as I
from hugectr_b200.ops import interaction_native as N

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,n,D", [(512, 27, 128), (1, 27, 128), (130, 9, 64), (77, 32, 128), (2048, 27, 32)])
def test_interaction_fwd_bwd(B, n, D):
    torch.manual_seed(0)
    mlp = (torch.randn(B, D, device="cuda") * 0.5).bfloat16()
    emb = (torch.randn(B, n - 1, D, device="cuda") * 0.5).bfloat16()
    w = D + n * (n - 1) // 2 + 1
    out = torch.full((B, w), 7.0, device="cuda", dtype=torch.bfloat16)
    assert N.available(mlp, emb, out)
    I.interaction_fwd(mlp, emb, out)
    ref = I.interaction_reference(mlp, emb)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 2e-2, err
    dout = (torch.randn(B, w, device="cuda") * 0.1).bfloat16()
    dmlp = torch.zeros_like(mlp)
    demb = torch.zeros_like(emb)
    I.interaction_bwd(mlp, emb, dout, dmlp, demb)
    m32 = mlp.float().requires_grad_(True)
    e32 = emb.float().requires_grad_(True)
    I.interaction_reference(m32, e32).backward(dout.float())
    torch.cuda.synchronize()
    for a, b in ((dmlp, m32.grad), (demb, e32.grad)):
        err = (a.float() - b).abs().max().item()
        assert err <= 3e-2 * b.abs().max().item() + 3e-2, err
