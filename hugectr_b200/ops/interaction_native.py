"""Loader shim for the sm_90a interaction kernel (csrc/interaction.cu)."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from . import dense as D

_ok = None


def _lib():
    global _ok
    l = _native.cuda_lib()
    if _ok is None:
        _ok = hasattr(l, "hctr_interaction_fwd")
        if _ok:
            vp, i = C.c_void_p, C.c_int
            l.hctr_interaction_fwd.argtypes = [vp, vp, vp, i, i, i, vp]
            l.hctr_interaction_bwd.argtypes = [vp, vp, vp, vp, vp, i, i, i, vp]
            l.hctr_interaction_fwd.restype = i
            l.hctr_interaction_bwd.restype = i
    return l


def available(mlp, emb, out, *grads) -> bool:
    """The kernels take contiguous bf16 tensors on 16-byte bases (they move rows in 16-byte vectors), n <= 32 and
    D <= 128, D % 16 == 0.  ``out`` is the forward's output or the backward's dout; ``grads`` the backward's
    dmlp and demb."""
    ts = (mlp, emb, out, *grads)
    if not (mlp.is_cuda and all(t.dtype == torch.bfloat16 for t in ts)):
        return False
    if not all(t.is_contiguous() and t.data_ptr() % 16 == 0 for t in ts):
        return False
    _lib()
    n = emb.shape[1] + 1
    return bool(_ok) and n <= 32 and mlp.shape[1] % 16 == 0 and mlp.shape[1] <= 128


def fwd(mlp, emb, out):
    rc = _lib().hctr_interaction_fwd(mlp.data_ptr(), emb.data_ptr(), out.data_ptr(), mlp.shape[0],
                                     emb.shape[1] + 1, mlp.shape[1],
                                     torch.cuda.current_stream().cuda_stream)
    if rc:
        raise RuntimeError("interaction_fwd failed")
    D._count()


def bwd(mlp, emb, dout, dmlp, demb):
    rc = _lib().hctr_interaction_bwd(mlp.data_ptr(), emb.data_ptr(), dout.data_ptr(),
                                     dmlp.data_ptr(), demb.data_ptr(), mlp.shape[0],
                                     emb.shape[1] + 1, mlp.shape[1],
                                     torch.cuda.current_stream().cuda_stream)
    if rc:
        raise RuntimeError("interaction_bwd failed")
    D._count()
