"""DLRM dot-product interaction (D2).

out[b] = [ mlp[b] (D) | strict lower triangle of X X^T, row-major (n(n-1)/2) | 0 ]  with
X = [mlp[b]; emb[b,0]; ...; emb[b,n-2]]  (reference HugeCTR/src/layers/interaction_layer.cu:47-274,
output width D + n(n-1)/2 + 1, :637).  The torch implementation below is the oracle and the CPU path;
the sm_90a kernel (csrc/interaction.cu) is used on GPU for bf16 when available.
"""
from __future__ import annotations

import torch

_tri_cache = {}


def _tri(n, device):
    k = (n, str(device))
    if k not in _tri_cache:
        idx = torch.tril_indices(n, n, -1, device=device)
        _tri_cache[k] = (idx[0], idx[1])
    return _tri_cache[k]


def interaction_reference(mlp, emb):
    b, d = mlp.shape
    x = torch.cat([mlp.unsqueeze(1), emb], dim=1).float()
    z = torch.bmm(x, x.transpose(1, 2))
    li, lj = _tri(x.shape[1], mlp.device)
    return torch.cat([mlp.float(), z[:, li, lj], torch.zeros(b, 1, device=mlp.device)], dim=1)


def interaction_fwd(mlp, emb, out):
    from . import interaction_native as N
    if N.available(mlp, emb, out):
        return N.fwd(mlp, emb, out)
    out.copy_(interaction_reference(mlp, emb).to(out.dtype))


def interaction_bwd(mlp, emb, dout, dmlp, demb):
    from . import interaction_native as N
    if dmlp is not None and demb is not None and N.available(mlp, emb, dout, dmlp, demb):
        return N.bwd(mlp, emb, dout, dmlp, demb)
    b, d = mlp.shape
    n = emb.shape[1] + 1
    x = torch.cat([mlp.unsqueeze(1), emb], dim=1).float()
    li, lj = _tri(n, mlp.device)
    g = dout.float()
    gz = torch.zeros(b, n, n, device=mlp.device)
    gz[:, li, lj] = g[:, d:d + li.numel()]
    gx = torch.bmm(gz + gz.transpose(1, 2), x)
    if dmlp is not None:
        dmlp.copy_((gx[:, 0] + g[:, :d]).to(dmlp.dtype))
    if demb is not None:
        demb.copy_(gx[:, 1:].to(demb.dtype))
