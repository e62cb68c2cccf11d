"""ctypes wrappers for csrc/dense_ops.cu with PyTorch fp32 fallbacks (CPU path == test oracle)."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from ..enums import Optimizer_t
from .optim import OPT_CODE, COptHyper, opt_hyper, opt_reference

EW_RELU, EW_RELU_BWD, EW_SIGMOID, EW_SIGMOID_BWD, EW_ADD, EW_SUB, EW_MUL, EW_SCALE, EW_ELU, \
    EW_ELU_BWD, EW_COPY, EW_ADD_INPLACE = range(12)

# short names of the element-wise rules that dense_opt_step takes
D_SGD, D_ADAGRAD, D_ADAM, D_FTRL, D_MOMENTUM, D_NESTEROV, D_RMSPROP = (
    Optimizer_t.SGD, Optimizer_t.AdaGrad, Optimizer_t.Adam, Optimizer_t.Ftrl, Optimizer_t.MomentumSGD,
    Optimizer_t.Nesterov, Optimizer_t.RMSProp)

launch_count = 0  # number of native kernel launches issued through this package


def _count(n=1):
    global launch_count
    launch_count += n


class DenseOptArgs(C.Structure):
    _fields_ = [("w", C.c_void_p), ("g", C.c_void_p), ("w16", C.c_void_p), ("s0", C.c_void_p),
                ("s1", C.c_void_p), ("n", C.c_longlong), ("hp", COptHyper), ("zero_grad", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        l = _native.cuda_lib()
        vp, ll, i, f = C.c_void_p, C.c_longlong, C.c_int, C.c_float
        l.hctr_dense_opt.argtypes = [C.POINTER(DenseOptArgs), i, vp]
        l.hctr_lr_step.argtypes = [vp, vp, f, f, f, C.c_uint, C.c_uint, C.c_uint, vp]
        l.hctr_bce_loss.argtypes = [vp, vp, vp, vp, i, f, f, i, i, i, vp]
        l.hctr_colsum.argtypes = [vp, vp, i, i, ll, i, vp]
        l.hctr_fc1_fwd.argtypes = [vp, vp, vp, vp, i, i, ll, i, i, vp]
        l.hctr_fc1_bwd.argtypes = [vp, vp, vp, vp, vp, vp, i, i, ll, ll, i, i, vp]
        l.hctr_copy2d.argtypes = [vp, vp, ll, i, ll, ll, i, i, vp]
        l.hctr_cast_pad.argtypes = [vp, vp, ll, i, i, ll, vp]
        l.hctr_elementwise.argtypes = [vp, vp, vp, ll, i, f, i, vp]
        l.hctr_cross_bwd_ew.argtypes = [vp, vp, vp, vp, vp, vp, i, i, i, i, i, vp]
        l.hctr_add3.argtypes = [vp, vp, vp, vp, ll, vp]
        for n in ("hctr_dense_opt", "hctr_lr_step", "hctr_bce_loss", "hctr_colsum", "hctr_fc1_fwd",
                  "hctr_fc1_bwd", "hctr_copy2d", "hctr_cast_pad", "hctr_elementwise",
                  "hctr_cross_bwd_ew", "hctr_add3"):
            getattr(l, n).restype = i
        if hasattr(l, "hctr_abi_size_dense_opt") and l.hctr_abi_size_dense_opt() != C.sizeof(DenseOptArgs):
            raise RuntimeError("libhctr_cuda.so DenseOptArgs layout differs from the python mirror: rebuild "
                               "the library (python -m hugectr_b200._native)")
        _lib = l
    return _lib


def _st(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _chk(rc, name):
    if rc != 0:
        raise RuntimeError(f"{name} failed rc={rc}")
    _count()


def _native_ok(*ts):
    return all(t is None or (t.is_cuda and t.dtype in (torch.float32, torch.bfloat16)) for t in ts) \
        and any(t is not None and t.is_cuda for t in ts)


def _isbf(t):
    return int(t.dtype == torch.bfloat16)


# ----------------------------------------------------------------------------- loss
def bce_loss(logits, labels, dx, loss_out, grad_scale, loss_scale, is_train, want_loss=True):
    """Fused BCE fwd + (train) grad / (eval) sigmoid written to dx (may alias logits).

    loss_out (fp32 [1]) += mean-loss contribution * loss_scale (loss_scale already includes 1/n).
    Semantics: reference HugeCTR/src/loss.cu:231-264.
    """
    n = logits.numel()
    if _native_ok(logits, dx) and labels.dtype == torch.float32:
        _chk(lib().hctr_bce_loss(logits.data_ptr(), labels.data_ptr(), dx.data_ptr(),
                                 loss_out.data_ptr(), n, float(grad_scale), float(loss_scale),
                                 int(is_train), int(want_loss), _isbf(logits), _st(logits)),
             "bce_loss")
        return
    x = logits.float().reshape(-1)
    y = labels.float().reshape(-1)
    if want_loss:
        l = torch.clamp(x, min=0) - x * y + torch.log1p(torch.exp(-x.abs()))
        loss_out.add_(l.sum() * loss_scale)
    sig = torch.sigmoid(x)
    res = (sig - y) * grad_scale if is_train else sig
    dx.copy_(res.reshape(dx.shape).to(dx.dtype))


# ----------------------------------------------------------------------------- reductions / skinny fc
def colsum_accum(x, out):
    """out[n] (fp32) += sum over rows of x[m, n]."""
    if _native_ok(x) and out.is_cuda and x.stride(1) == 1:
        _chk(lib().hctr_colsum(x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], x.stride(0),
                               _isbf(x), _st(x)), "colsum")
        return
    out.add_(x.float().sum(0))


def fc1_fwd(x, w, b, y, relu=False):
    """y[m] = act(x[m,:] . w + b) for num_output == 1 layers (w fp32 [K])."""
    if _native_ok(x, y) and x.stride(1) == 1:
        _chk(lib().hctr_fc1_fwd(x.data_ptr(), w.data_ptr(), 0 if b is None else b.data_ptr(),
                                y.data_ptr(), x.shape[0], x.shape[1], x.stride(0), int(relu),
                                _isbf(x), _st(x)), "fc1_fwd")
        return
    K = w.numel()          # x may be the zero-padded staging copy (K rounded up to 8 in mixed precision)
    v = x[:, :K].float() @ w.float().reshape(-1, 1)
    if b is not None:
        v = v + b.float()
    if relu:
        v = torch.relu(v)
    y.copy_(v.reshape(y.shape).to(y.dtype))


def fc1_bwd(x, w, dy, dx, dw, db, mask_relu=False):
    """dx = dy (x) w (masked by x>0 when mask_relu); dw += x^T dy; db += sum(dy)."""
    if _native_ok(x, dy) and x.stride(1) == 1 and (dx is None or dx.stride(1) == 1):
        _chk(lib().hctr_fc1_bwd(x.data_ptr(), w.data_ptr(), dy.data_ptr(),
                                0 if dx is None else dx.data_ptr(), dw.data_ptr(),
                                0 if db is None else db.data_ptr(), x.shape[0], x.shape[1],
                                x.stride(0), 0 if dx is None else dx.stride(0), int(mask_relu),
                                _isbf(x), _st(x)), "fc1_bwd")
        return
    g = dy.float().reshape(-1, 1)
    K = w.numel()
    xk = x[:, :K].float()
    dw.add_((xk * g).sum(0).reshape(dw.shape))
    if db is not None:
        db.add_(g.sum().reshape(db.shape))
    if dx is not None:
        d = g * w.float().reshape(1, -1)
        if mask_relu:
            d = d * (xk > 0)
        if dx.shape[1] > K:
            dx[:, K:].zero_()
        dx[:, :K].copy_(d.to(dx.dtype))


# ----------------------------------------------------------------------------- copies / casts
def copy2d(src, dst, accumulate=False):
    """dst[r, c] (+)= src[r, c] for 2-D (possibly strided) views with unit inner stride."""
    assert src.shape == dst.shape and src.dim() == 2
    if (_native_ok(src, dst) and src.dtype == dst.dtype and src.stride(1) == 1
            and dst.stride(1) == 1):
        _chk(lib().hctr_copy2d(src.data_ptr(), dst.data_ptr(), src.shape[0], src.shape[1],
                               src.stride(0), dst.stride(0), src.element_size(), int(accumulate),
                               _st(src)), "copy2d")
        return
    if accumulate:
        dst.add_(src.to(dst.dtype))
    else:
        dst.copy_(src)


def cast_pad(src, dst):
    """fp32 [M,K] -> bf16 [M,Kp] zero padded (TMA needs 16-byte row pitch)."""
    if src.is_cuda and src.dtype == torch.float32 and dst.dtype == torch.bfloat16 \
            and src.stride(1) == 1 and dst.is_contiguous():
        _chk(lib().hctr_cast_pad(src.data_ptr(), dst.data_ptr(), src.shape[0], src.shape[1],
                                 dst.shape[1], src.stride(0), _st(src)), "cast_pad")
        return
    dst.zero_()
    dst[:, :src.shape[1]].copy_(src.to(dst.dtype))


def elementwise(op, a, b, out, alpha=0.0):
    if _native_ok(a, b, out) and a.is_contiguous() and out.is_contiguous() and \
            (b is None or (b.is_contiguous() and b.dtype == a.dtype)) and a.dtype == out.dtype:
        _chk(lib().hctr_elementwise(a.data_ptr(), 0 if b is None else b.data_ptr(), out.data_ptr(),
                                    a.numel(), op, float(alpha), _isbf(a), _st(a)), "elementwise")
        return
    x = a.float()
    y = None if b is None else b.float()
    if op == EW_RELU: r = torch.relu(x)
    elif op == EW_RELU_BWD: r = x * (y > 0)
    elif op == EW_SIGMOID: r = torch.sigmoid(x)
    elif op == EW_SIGMOID_BWD: r = x * y * (1 - y)
    elif op == EW_ADD: r = x + y
    elif op == EW_SUB: r = x - y
    elif op == EW_MUL: r = x * y
    elif op == EW_SCALE: r = x * alpha
    elif op == EW_ELU: r = torch.where(x > 0, x, alpha * (torch.exp(x) - 1))
    elif op == EW_ELU_BWD: r = torch.where(y > 0, x, x * (y + alpha))
    elif op == EW_ADD_INPLACE: r = out.float() + x
    else: r = x
    out.copy_(r.to(out.dtype))


def cross_bwd_ew(dy, x0, t, dt, dx0, first, db=None, last=False, row_splits=0):
    """dt = dy*x0 ; dx0 = (0 if first else dx0) + dy*t (+ dy if last) ; db (fp32 [cols]) += colsum(dt).
    dx0 is fp32 or bf16 (accumulated in fp32 registers either way)."""
    if _native_ok(dy, x0, t, dt) and dy.dtype == torch.bfloat16 and dy.is_contiguous() \
            and x0.is_contiguous() and t.is_contiguous() and dy.shape[-1] % 8 == 0:
        rows, cols = dy.shape[0], dy.shape[1]
        _chk(lib().hctr_cross_bwd_ew(dy.data_ptr(), x0.data_ptr(), t.data_ptr(), dt.data_ptr(),
                                     dx0.data_ptr(), 0 if db is None else db.data_ptr(), rows, cols,
                                     int(bool(first)) | (2 if last else 0),
                                     int(dx0.dtype == torch.bfloat16), int(row_splits), _st(dy)),
             "cross_bwd_ew")
        return
    d = dy.float()
    dtv = (d * x0.float()).to(dt.dtype)
    dt.copy_(dtv)
    if db is not None:
        db.add_(dtv.float().sum(0))
    acc = d * t.float() + (d if last else 0.0)
    if first:
        dx0.copy_(acc.to(dx0.dtype))
    else:
        dx0.copy_((dx0.float() + acc).to(dx0.dtype))


def partial_sum(part, out2d, col0, k, w):
    """out2d[:, col0:col0+w] = part.view(rows, k, w).sum(1)  (partials of a row-sharded table)"""
    rows = out2d.shape[0]
    if _native_ok(part, out2d) and part.dtype == out2d.dtype and part.is_contiguous() \
            and part.dtype in (torch.bfloat16, torch.float32) and out2d.stride(1) == 1:
        l = lib()
        if not hasattr(l, "_ps_ready"):
            l.hctr_partial_sum.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_longlong, C.c_int, C.c_int, C.c_void_p]
            l.hctr_partial_sum.restype = C.c_int
            l._ps_ready = True
        _chk(l.hctr_partial_sum(part.data_ptr(), out2d.data_ptr(), rows, k, w, out2d.stride(0), col0,
                                int(part.dtype == torch.bfloat16), _st(part)), "partial_sum")
        return
    out2d[:, col0:col0 + w] = part.reshape(rows, k, w).float().sum(1).to(out2d.dtype)


def add3(a, b, c, out):
    """out = a + b (+ c fp32)."""
    if _native_ok(a, b, out) and a.dtype == torch.bfloat16 and a.is_contiguous() and \
            b.is_contiguous() and out.is_contiguous() and a.numel() % 8 == 0:
        _chk(lib().hctr_add3(a.data_ptr(), b.data_ptr(), 0 if c is None else c.data_ptr(),
                             out.data_ptr(), a.numel(), _st(a)), "add3")
        return
    r = a.float() + b.float()
    if c is not None:
        r = r + c
    out.copy_(r.to(out.dtype))


# ----------------------------------------------------------------------------- optimizers
def dense_opt_step(opt, w, g, w16, s0, s1, lr_t, step_t, hp, zero_grad=True):
    """One fused launch over the flat arena with the element-wise rule of ``opt`` (an Optimizer_t).
    hp: dict of hyper-parameters (optim.opt_hp)."""
    if w.is_cuda:
        a = DenseOptArgs(w.data_ptr(), g.data_ptr(), 0 if w16 is None else w16.data_ptr(),
                         0 if s0 is None else s0.data_ptr(), 0 if s1 is None else s1.data_ptr(),
                         w.numel(), opt_hyper(hp, lr_t, step_t), int(zero_grad))
        _chk(lib().hctr_dense_opt(C.byref(a), OPT_CODE[opt], _st(w)), "dense_opt")
        return
    dense_opt_reference(opt, w, g, w16, s0, s1, float(lr_t.item()), int(step_t.item()), hp, zero_grad)


def dense_opt_reference(opt, w, g, w16, s0, s1, lr, step, hp, zero_grad=True):
    """fp32 PyTorch implementation of the Appendix A.2 update rules (oracle + CPU path)."""
    opt_reference(opt, w, s0, s1, g, hp, lr, step)
    if w16 is not None:
        w16.copy_(w.to(w16.dtype))
    if zero_grad:
        g.zero_()


def lr_step(step_t, lr_t, base_lr, end_lr, decay_power, warmup, decay_start, decay_steps):
    """Advance the device-side step counter and learning rate (Appendix A.5 schedule)."""
    if step_t.is_cuda:
        _chk(lib().hctr_lr_step(step_t.data_ptr(), lr_t.data_ptr(), float(base_lr), float(end_lr),
                                float(decay_power), int(warmup), int(decay_start), int(decay_steps),
                                _st(step_t)), "lr_step")
        return
    from ..lr_scheduler import lr_at
    t = int(step_t.item()) + 1
    step_t.fill_(t)
    lr_t.fill_(lr_at(t, base_lr, warmup, decay_start, decay_steps, decay_power, end_lr))
