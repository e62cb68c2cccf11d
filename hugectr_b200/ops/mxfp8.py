"""Block-scaled (OCP MX) fp8 GEMM: ctypes bindings for csrc/gemm_mxfp8.cu + a PyTorch reference.

Format: e4m3 values, one UE8M0 (power-of-two) scale per 32 consecutive elements along K.  Scales are stored in the
512-byte block layout the tensor core copy wants (see the kernel file): ``sf[(r // 128) * (K // 128) + k // 128]``
is a [32, 4, 4] byte block indexed ``[r % 32][(r % 128) // 32][(k % 128) // 32]``.
"""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from . import dense as D
from . import gemm as G

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = _native.cuda_lib()
        vp, i, ll, f = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        l.hctr_mx_quantize.argtypes = [vp, ll, vp, vp, i, i, i, i, vp]
        l.hctr_gemm_mxfp8.argtypes = [vp, vp, vp, vp, vp, i, i, i, ll, vp, f, i, vp]
        l.hctr_mx_quantize.restype = l.hctr_gemm_mxfp8.restype = i
        _lib = l
    return _lib


def _pad128(n: int) -> int:
    return (n + 127) // 128 * 128


def mx_buffers(rows: int, cols: int, device):
    """(q uint8 [rows_pad, cols], sf uint8 [(rows_pad / 128) * (cols / 128) * 512])"""
    rp = _pad128(rows)
    return (torch.empty(rp, cols, dtype=torch.uint8, device=device),
            torch.empty((rp // 128) * (cols // 128) * 512, dtype=torch.uint8, device=device))


def mx_quantize(x: torch.Tensor, q=None, sf=None, transposed: bool = False):
    """x [rows, cols] (bf16 / fp32; ``transposed``: x is stored [cols, rows]) -> (q, sf).  cols % 128 == 0."""
    rows, cols = (x.shape[1], x.shape[0]) if transposed else x.shape
    assert cols % 128 == 0, "MX quantisation works on K blocks of 128"
    if q is None:
        q, sf = mx_buffers(rows, cols, x.device)
    if x.is_cuda:
        assert x.stride(1) == 1
        rc = lib().hctr_mx_quantize(x.data_ptr(), x.stride(0), q.data_ptr(), sf.data_ptr(), rows, cols,
                                    int(x.dtype == torch.bfloat16), int(transposed),
                                    torch.cuda.current_stream(x.device).cuda_stream)
        if rc:
            raise RuntimeError(f"hctr_mx_quantize failed rc={rc}")
        D._count()
        return q, sf
    qr, sfr = mx_quantize_reference(x.t() if transposed else x)
    q.copy_(qr)
    sf.copy_(sfr)
    return q, sf


def e4m3_scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """fp32 exponents e of the power-of-two scales of blocks whose largest magnitudes are ``amax`` (fp32, >= 0): the
    smallest 2^e with amax / 2^e <= 448 (e4m3 max), clamped to [-127, 127], -127 for amax == 0 -- computed as
    e4m3_scale_exp in csrc/ptx.cuh, from the bits of amax = m * 2^ex: e = ex - 9 + (m > 0.875)"""
    b = amax.to(torch.float32).contiguous().view(torch.int32)
    e = (b >> 23) - 135 + ((b & 0x7FFFFF) > 0x600000).to(torch.int32)
    return torch.where(b < 0x00800000, -127, e).clamp(-127, 127).to(torch.float32)


def mx_quantize_reference(x: torch.Tensor):
    rows, cols = x.shape
    rp = _pad128(rows)
    xf = torch.zeros(rp, cols, dtype=torch.float32)
    xf[:rows] = x.float().cpu()
    blk = xf.view(rp, cols // 32, 32)
    e = e4m3_scale_exponent(blk.abs().amax(-1))
    qv = (blk * torch.ldexp(torch.ones_like(e), (-e).to(torch.int32)).unsqueeze(-1)).reshape(rp, cols).to(torch.float8_e4m3fn)
    q = qv.view(torch.uint8)
    sfb = (e + 127).to(torch.uint8)                                   # [rp, cols / 32]
    # block layout: [rp/128][cols/128][32][4][4] <- [r%32][(r%128)//32][k]
    t = sfb.view(rp // 128, 4, 32, cols // 128, 4)                    # (R, j, i, KB, k)
    sf = t.permute(0, 3, 2, 1, 4).contiguous().reshape(-1)
    return q, sf


def mx_dequantize(q: torch.Tensor, sf: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
    rp = q.shape[0]
    v = q.cpu().view(torch.float8_e4m3fn).float().view(rp, cols // 32, 32)
    t = sf.cpu().view(rp // 128, cols // 128, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(rp, cols // 32)
    return (v * torch.exp2(t.float() - 127.0).unsqueeze(-1)).reshape(rp, cols)[:rows]


GEMM_FLAGS = G.EPI_RELU | G.EPI_SIGMOID | G.EPI_OUT_F32


def gemm_mxfp8_eligible(aq, sfa, bq, sfb, M: int, N: int, K: int, out, bias=None, flags: int = 0) -> bool:
    """What hctr_gemm_mxfp8 reads and writes is there: the epilogue flags it implements (the others read
    tensors it is not given), q / sf buffers as large as the tensor maps and the scale bulk copies cover
    (contiguous, 16-byte bases), and an ``out`` / ``bias`` the epilogue can address with its 16-byte
    vector loads and stores (``gemm.epi_eligible``)."""
    if flags & ~GEMM_FLAGS or K <= 0 or K % 128:
        return False
    mp, np_ = _pad128(M), _pad128(N)
    for t, need in ((aq, mp * K), (bq, np_ * K), (sfa, mp // 128 * (K // 128) * 512),
                    (sfb, np_ // 128 * (K // 128) * 512)):
        if t.element_size() != 1 or not t.is_contiguous() or t.numel() < need or t.data_ptr() % 16:
            return False
    want = torch.float32 if flags & G.EPI_OUT_F32 else torch.bfloat16
    if out.dtype != want or out.dim() != 2 or out.shape[0] < M or out.shape[1] < N:
        return False
    if bias is not None and (bias.dtype != torch.float32 or bias.numel() < N):
        return False
    return G.epi_eligible(M, N, out, bias)


def gemm_mxfp8(aq, sfa, bq, sfb, M: int, N: int, K: int, out=None, bias=None, flags: int = 0, alpha: float = 1.0):
    """out[M, N] = epilogue(alpha * deq(A)[M, K] @ deq(B)[N, K]^T (+ bias)); flags: EPI_RELU, EPI_SIGMOID,
    EPI_OUT_F32.  Raises ValueError, before any launch, on arguments gemm_mxfp8_eligible rejects."""
    f32 = bool(flags & G.EPI_OUT_F32)
    if out is None:
        out = torch.empty(M, N, device=aq.device, dtype=torch.float32 if f32 else torch.bfloat16)
    if aq.is_cuda:
        if not gemm_mxfp8_eligible(aq, sfa, bq, sfb, M, N, K, out, bias, flags):
            raise ValueError(f"gemm_mxfp8: M={M} N={N} K={K} flags={flags}: unsupported flags, undersized or "
                             "misaligned q / sf buffers, or an out / bias the epilogue cannot address")
        rc = lib().hctr_gemm_mxfp8(aq.data_ptr(), sfa.data_ptr(), bq.data_ptr(), sfb.data_ptr(), out.data_ptr(), M, N,
                                   K, out.stride(0), 0 if bias is None else bias.data_ptr(), float(alpha), int(flags),
                                   torch.cuda.current_stream(aq.device).cuda_stream)
        if rc:
            raise RuntimeError(f"hctr_gemm_mxfp8 failed rc={rc}")
        D._count()
        return out
    v = mx_dequantize(aq, sfa, M, K) @ mx_dequantize(bq, sfb, N, K).t() * alpha
    if bias is not None:
        v = v + bias.float()
    if flags & G.EPI_RELU:
        v = torch.relu(v)
    out.copy_(v.to(out.dtype))
    return out
