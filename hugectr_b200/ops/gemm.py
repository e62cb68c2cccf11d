"""bf16 tensor-core GEMM with fused epilogues (wgmma/TMA kernel in csrc/gemm_tc.cu).

``gemm_bf16`` is the single entry point used by the MLP / InnerProduct / MultiCross layers for
fprop, dgrad and wgrad.  On CPU (or for shapes TMA cannot address) it falls back to an fp32
PyTorch reference that implements exactly the same epilogue math; the same function is the
numerics oracle in the tests.
"""
from __future__ import annotations

import ctypes

import torch

from .. import _native

EPI_RELU = 1
EPI_OUT_F32 = 2
EPI_ATOMIC = 4
EPI_CROSS = 16
EPI_MASK = 32
EPI_SIGMOID = 64
EPI_ADD = 128

_c = ctypes
_sig_set = False


def _lib():
    global _sig_set
    lib = _native.cuda_lib()
    if not _sig_set:
        lib.hctr_gemm_bf16.restype = _c.c_int
        lib.hctr_gemm_bf16.argtypes = [
            _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int,
            _c.c_longlong, _c.c_longlong, _c.c_longlong, _c.c_int, _c.c_int,
            _c.c_void_p, _c.c_void_p, _c.c_longlong, _c.c_void_p, _c.c_void_p, _c.c_longlong,
            _c.c_void_p, _c.c_longlong, _c.c_float, _c.c_int, _c.c_int, _c.c_int, _c.c_void_p]
        _sig_set = True
    return lib


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def tc_eligible(a: torch.Tensor, b: torch.Tensor, a_mn: bool, b_mn: bool) -> bool:
    """TMA needs 16-byte aligned bases and row pitches; the wgmma path is bf16 only."""
    if not (a.is_cuda and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16):
        return False
    for t in (a, b):
        if t.dim() != 2 or t.stride(1) != 1 or (t.stride(0) * 2) % 16 or t.data_ptr() % 16:
            return False
    return True


def epi_eligible(M: int, N: int, out, bias=None, mask=None, x0=None, xl=None, aux=None) -> bool:
    """The kernel's epilogue reads and writes its tensors row-major with unit column stride, and from N >= 32 on in
    16-byte vectors or TMA boxes at every 32-column chunk of a row: 16-byte bases and row pitches.  x0 and xl
    share one pitch."""
    for t in (out, mask, x0, xl, aux):
        if t is None:
            continue
        if t.dim() != 2 or t.stride(1) != 1:
            return False
        if N >= 32 and (t.data_ptr() % 16 or (M > 1 and (t.stride(0) * t.element_size()) % 16)):
            return False
    if bias is not None and ((N > 1 and bias.stride(-1) != 1) or (N >= 32 and bias.data_ptr() % 16)):
        return False
    if x0 is not None and xl is not None and x0.stride(0) != xl.stride(0):
        return False
    return True


def gemm_reference(a, b, a_mn=False, b_mn=False, bias=None, mask=None, x0=None, xl=None,
                   alpha=1.0, flags=0, out=None, aux=None):
    """fp32 PyTorch oracle with the same epilogue semantics as the kernel."""
    A = a.float().t() if a_mn else a.float()          # [M, K]
    B = b.float() if b_mn else b.float().t()          # [K, N]
    v = (A @ B) * alpha
    if bias is not None:
        v = v + bias.float()
    if flags & EPI_CROSS:
        if aux is not None:
            aux.copy_(v.to(aux.dtype))
        v = x0.float() * v + xl.float()
    if flags & EPI_ADD:
        v = v + xl.float()
    if flags & EPI_MASK:
        v = v * (mask.float() > 0)
    if flags & EPI_RELU:
        v = torch.relu(v)
    if flags & EPI_SIGMOID:
        v = torch.sigmoid(v)
    if flags & EPI_ATOMIC:
        out.add_(v.to(out.dtype))
        return out
    odt = torch.float32 if (flags & EPI_OUT_F32) else a.dtype
    if out is None:
        return v.to(odt)
    out.copy_(v.to(out.dtype))
    return out


_bn_override = {}

# "tc": the hand-written wgmma kernels (product path).  "library": bf16 GEMMs through torch.mm
# (cuBLAS / cuBLASLt) with eager epilogues -- the stand-in baseline arm of bench.py, never a default.
IMPL = "tc"
_fallback_logged = set()


def set_impl(name: str):
    global IMPL
    assert name in ("tc", "library")
    IMPL = name


def gemm_library(a, b, a_mn=False, b_mn=False, bias=None, mask=None, x0=None, xl=None,
                 alpha=1.0, flags=0, out=None, aux=None):
    """Same contract as ``gemm_reference`` with the matmul in the operands' dtype on the vendor
    library (what a cuBLASLt-based framework runs): bias through addmm, the rest eager."""
    A = a.t() if a_mn else a
    B = b if b_mn else b.t()
    f32 = bool(flags & (EPI_OUT_F32 | EPI_ATOMIC))
    if f32:
        v = torch.mm(A, B).float()
        if alpha != 1.0:
            v = v * alpha
        if bias is not None:
            v = v + bias.float()
    elif bias is not None and alpha == 1.0:
        v = torch.addmm(bias.to(A.dtype), A, B)
    else:
        v = torch.mm(A, B)
        if alpha != 1.0:
            v = v * alpha
        if bias is not None:
            v = v + bias.to(v.dtype)
    if flags & EPI_CROSS:
        if aux is not None:
            aux.copy_(v)
        v = torch.addcmul(xl.to(v.dtype), x0.to(v.dtype), v)
    if flags & EPI_ADD:
        v = v + xl.to(v.dtype)
    if flags & EPI_MASK:
        v = v * (mask > 0).to(v.dtype)
    if flags & EPI_RELU:
        v = torch.relu(v)
    if flags & EPI_SIGMOID:
        v = torch.sigmoid(v)
    if flags & EPI_ATOMIC:
        out.add_(v.to(out.dtype))
        return out
    if out is None:
        return v
    out.copy_(v)
    return out


def _pick_block_n(M, N, K, splits):
    """Tile / cluster choice.  1000 + BN selects the 2-CTA cluster kernel: the two CTAs take adjacent 128-row
    tiles and multicast the shared B tile (halves the L2->SM traffic of B)."""
    import os
    ov = os.environ.get("HCTR_GEMM_BN")
    if ov:
        return int(ov)
    if N <= 64:
        return 64
    m_t = (M + 127) // 128
    if m_t < 2:
        return 128
    # the 256-wide tile reads A half as often per MAC but loses when it costs an extra wave of the
    # 66 cluster pairs of an H100 (132 SMs); the autotuner below times both on first sight of a shape
    def waves(bn):
        items = ((m_t + 1) // 2) * ((N + bn - 1) // bn) * max(1, splits)
        return (items + 65) // 66
    if N >= 256 and waves(256) * 2 * 0.88 <= waves(128):
        return 1256
    return 1128


def gemm_bf16(a, b, out=None, *, a_mn=False, b_mn=False, bias=None, mask=None, x0=None, xl=None,
              aux=None, alpha=1.0, flags=0, splits=1, block_n=0, colsum=None):
    """out[M,N] = epilogue(alpha * op(a) @ op(b)).

    ``colsum`` (fp32 [N], optional): += column sums of the bf16 output, i.e. the bias gradient of the
    layer that consumes ``out`` as its dY (one reduction kernel after the GEMM).

    a: ``[M,K]`` (K-major) or ``[K,M]`` when ``a_mn``;  b: ``[N,K]`` or ``[K,N]`` when ``b_mn``.
    """
    M = a.shape[1] if a_mn else a.shape[0]
    K = a.shape[0] if a_mn else a.shape[1]
    N = b.shape[1] if b_mn else b.shape[0]
    f32_out = bool(flags & (EPI_OUT_F32 | EPI_ATOMIC))
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.float32 if f32_out else a.dtype)
    if IMPL == "library" and a.is_cuda:
        r = gemm_library(a, b, a_mn, b_mn, bias, mask, x0, xl, alpha, flags, out, aux)
        if colsum is not None:
            colsum.add_(out.float().sum(0))
        return r
    operands_ok = tc_eligible(a, b, a_mn, b_mn)
    if not operands_ok or not epi_eligible(M, N, out, bias, mask, x0, xl, aux):
        if a.is_cuda:
            # never silent: a misaligned / non-bf16 operand or epilogue tensor moves this GEMM off the wgmma kernel
            sig = (M, N, K, str(a.dtype), tuple(a.stride()), tuple(b.stride()), a.data_ptr() % 16,
                   b.data_ptr() % 16, operands_ok)
            if sig not in _fallback_logged:
                _fallback_logged.add(sig)
                from ..utils import logger
                what = (f"an epilogue tensor (out / bias / mask / x0 / xl / aux, flags={flags})" if operands_ok
                        else f"dtype={a.dtype} strides a={tuple(a.stride())} b={tuple(b.stride())}")
                logger.warning(f"gemm_bf16: M={M} N={N} K={K} {what} is not TMA-addressable (16-byte base / pitch, "
                               "bf16): running the library matmul instead of the wgmma kernel")
        r = gemm_reference(a, b, a_mn, b_mn, bias, mask, x0, xl, alpha, flags, out, aux)
        if colsum is not None:
            colsum.add_(out.float().sum(0))
        return r
    if splits > 1:
        flags |= EPI_ATOMIC
    if block_n == 0:
        block_n = _tuned_block_n(a, b, out, M, N, K, a_mn, b_mn, bias, mask, x0, xl, aux, alpha, flags, splits)
    _launch(a, b, out, M, N, K, a_mn, b_mn, bias, mask, x0, xl, aux, alpha, flags, splits, block_n)
    if colsum is not None:
        from . import dense as _D
        _D.colsum_accum(out, colsum)
    return out


def _launch(a, b, out, M, N, K, a_mn, b_mn, bias, mask, x0, xl, aux, alpha, flags, splits, block_n):
    stream = torch.cuda.current_stream(a.device).cuda_stream
    args = [a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0),
            out.stride(0), int(a_mn), int(b_mn), _ptr(bias), _ptr(mask),
            0 if mask is None else mask.stride(0), _ptr(x0), _ptr(xl),
            0 if xl is None else xl.stride(0), _ptr(aux), 0 if aux is None else aux.stride(0),
            float(alpha), int(flags), int(splits), int(block_n), stream]
    rc = _lib().hctr_gemm_bf16(*args)
    if rc != 0:
        raise RuntimeError(f"hctr_gemm_bf16 failed rc={rc} M={M} N={N} K={K}")
    from . import dense as _D
    _D._count()


# ----------------------------------------------------------------------------- tile autotuner
# The analogue of the reference's cublasLt algorithm search (GemmFunctor::search_algorithm,
# HugeCTR/src/layers/functors/fused_fc_layer_functors.cu: 16 heuristics x 100 repetitions at
# initialisation): the first time a (shape, layout, epilogue) is seen outside graph capture, the
# candidate tile configurations are timed on scratch outputs and the fastest is cached.
_TUNE_CACHE = {}


def _tuned_block_n(a, b, out, M, N, K, a_mn, b_mn, bias, mask, x0, xl, aux, alpha, flags, splits):
    import os
    heur = _pick_block_n(M, N, K, splits)
    if heur < 1000 or os.environ.get("HCTR_GEMM_AUTOTUNE", "1") == "0" or os.environ.get("HCTR_GEMM_BN"):
        return heur
    key = (M, N, K, bool(a_mn), bool(b_mn), int(flags), int(splits), out.dtype, out.stride(0),
           aux is not None, bias is not None)
    hit = _TUNE_CACHE.get(key)
    if hit is not None:
        return hit
    if torch.cuda.is_current_stream_capturing():
        return heur
    cands = [1128, 1256] if N >= 256 else [1128]
    if not (flags & (EPI_OUT_F32 | EPI_ATOMIC)):
        # with the TMA epilogue, memory-bound bf16-output calls can win on more, narrower tiles
        cands = [1064] + cands + [64, 128, 256]
    if len(cands) == 1:
        _TUNE_CACHE[key] = cands[0]
        return cands[0]
    so = torch.empty_strided(out.size(), out.stride(), dtype=out.dtype, device=out.device)
    if flags & EPI_ATOMIC:
        so.zero_()
    sa = (torch.empty_strided(aux.size(), aux.stride(), dtype=aux.dtype, device=aux.device)
          if aux is not None else None)
    for bn in cands:
        for _ in range(2):
            _launch(a, b, so, M, N, K, a_mn, b_mn, bias, mask, x0, xl, sa, alpha, flags, splits, bn)
    # candidates alternate over the rounds so that a slow spell of a shared GPU does not decide the pick
    times = {bn: [] for bn in cands}
    for _ in range(3):
        for bn in cands:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                _launch(a, b, so, M, N, K, a_mn, b_mn, bias, mask, x0, xl, sa, alpha, flags, splits, bn)
            e1.record()
            e1.synchronize()
            times[bn].append(e0.elapsed_time(e1))
    best = min(cands, key=lambda bn: sorted(times[bn])[1])
    _TUNE_CACHE[key] = best
    return best
