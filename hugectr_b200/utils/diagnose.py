"""Debug helpers: NaN/Inf verification, histogram and sampling of tensors, kernel timing.

Parity: HugeCTR/src/diagnose.cu:45-208 (verify / histogram / sample),
HugeCTR/include/base/debug/cuda_debugging.hpp:44-96 (HCTR_CUDA_KERNEL_TIME / _SUMMARY).
"""
from __future__ import annotations

import contextlib
import time

import torch

from . import logger


def verify(tensor: torch.Tensor, name: str = "tensor", raise_on_error: bool = True) -> bool:
    """True when the tensor has no NaN/Inf (diagnose::verify_and_histogram)."""
    t = tensor.detach().float()
    bad = int((~torch.isfinite(t)).sum().item())
    if bad:
        msg = f"{name}: {bad} non-finite values out of {t.numel()}"
        if raise_on_error:
            raise RuntimeError(msg)
        logger.error(msg)
        return False
    return True


def histogram(tensor: torch.Tensor, bins: int = 16, name: str = "tensor") -> torch.Tensor:
    t = tensor.detach().float().reshape(-1)
    lo, hi = float(t.min()), float(t.max())
    h = torch.histc(t, bins=bins, min=lo, max=hi if hi > lo else lo + 1)
    logger.info(f"{name}: min {lo:.6g} max {hi:.6g} hist {h.int().tolist()}")
    return h


def sample(tensor: torch.Tensor, n: int = 16, name: str = "tensor") -> torch.Tensor:
    t = tensor.detach().reshape(-1)
    idx = torch.linspace(0, t.numel() - 1, min(n, t.numel())).long().to(t.device)
    s = t[idx].float().cpu()
    logger.info(f"{name}: samples {[round(float(x), 6) for x in s]}")
    return s


def verify_model(model) -> bool:
    """NaN scan over weights, wgrads and every activation of the training graph."""
    ok = verify(model.arena.weights, "dense weights", False)
    ok &= verify(model.arena.wgrad, "dense wgrad", False)
    for name, t in model.net_train.tensors.items():
        if t.data is not None and t.data.dtype.is_floating_point:
            ok &= verify(t.data, name, False)
    return ok


@contextlib.contextmanager
def kernel_time(name: str, iters: int = 1):
    """Device-timed region (CUDA events on the current stream) -- HCTR_CUDA_KERNEL_TIME."""
    if torch.cuda.is_available():
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        yield
        e.record()
        torch.cuda.synchronize()
        logger.info(f"[time] {name}: {s.elapsed_time(e) / iters * 1000:.1f} us")
    else:
        t0 = time.perf_counter()
        yield
        logger.info(f"[time] {name}: {(time.perf_counter() - t0) / iters * 1e6:.1f} us")


def nvtx_range(name: str):
    """NVTX range context (reference only annotates data-reader threads, data_collector.cpp:124)."""
    if torch.cuda.is_available():
        return torch.cuda.nvtx.range(name)
    return contextlib.nullcontext()


def kernel_summary(pattern: str = "", log: bool = False):
    """Static resources of every kernel in lib/libhctr_cuda.so -- the role of HCTR_CUDA_KERNEL_SUMMARY
    (registers / shared memory / occupancy from cudaFuncGetAttributes, cuda_debugging.hpp:44-70),
    read from the cubin with ``cuobjdump -res-usage`` so that it also works without a GPU.
    Returns {demangled kernel name: {"regs", "smem", "stack", "local", "max_blocks_per_sm"}}; the
    occupancy bound is the register / static-shared-memory limit of sm_90 (64 K registers, 227 KB
    shared memory, 2048 threads per SM) for a 256-thread block."""
    import re
    import shutil
    import subprocess
    from .. import _native
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([exe, "-res-usage", _native.CUDA_SO], capture_output=True, text=True).stdout
    names = re.findall(r"Function (\S+):\n\s+(.*)", out)
    filt = shutil.which("c++filt")
    dem = {}
    if filt and names:
        r = subprocess.run([filt], input="\n".join(n for n, _ in names), capture_output=True, text=True).stdout
        dem = dict(zip([n for n, _ in names], r.split("\n")))
    res = {}
    for sym, line in names:
        f = dict(kv.split(":") for kv in re.findall(r"[A-Z]+:\d+", line))
        regs, smem = int(f.get("REG", 0)), int(f.get("SHARED", 0))
        name = dem.get(sym, sym)
        if pattern and pattern not in name:
            continue
        by_regs = 65536 // max(1, regs * 256)
        by_smem = (227 * 1024) // smem if smem else 32
        res[name] = {"regs": regs, "smem": smem, "stack": int(f.get("STACK", 0)), "local": int(f.get("LOCAL", 0)),
                     "max_blocks_per_sm": max(0, min(8, by_regs, by_smem))}
        if log:
            logger.info(f"[kernel] {name.split('(')[0][:80]}: {regs} regs, {smem} B static smem, "
                        f"{f.get('STACK', 0)} B stack")
    return res
