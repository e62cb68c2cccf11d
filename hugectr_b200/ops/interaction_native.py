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


def available(mlp, emb, out) -> bool:
    if not (mlp.is_cuda and mlp.dtype == torch.bfloat16 and emb.dtype == torch.bfloat16
            and out.dtype == torch.bfloat16):
        return False
    if not (mlp.is_contiguous() and emb.is_contiguous() and out.is_contiguous()):
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
