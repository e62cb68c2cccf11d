"""Native code build + loader.

All device code lives in ``hugectr_b200/csrc/*.cu`` and is compiled **only** for sm_90a
(``-gencode arch=compute_90a,code=sm_90a``, the H100) into ``hugectr_b200/lib/libhctr_cuda.so``; host-side
native runtime pieces (readers, generators, host parameter server, thread pool) live in
``csrc/host/*.cpp`` -> ``lib/libhctr_host.so``.  Launchers are ``extern "C"`` and are called through
ctypes with raw device pointers and the current torch CUDA stream, so the kernels run on torch's
streams and are captured by CUDA graphs like any other launch.

The shared objects are built in-tree (git-ignored) by ``build()``.
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIBDIR = os.path.join(_HERE, "lib")
CUDA_SO = os.path.join(LIBDIR, "libhctr_cuda.so")
HOST_SO = os.path.join(LIBDIR, "libhctr_host.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-pthread", "-fopenmp", "-march=x86-64-v3"]

_lock = threading.Lock()
_cuda_lib = None
_host_lib = None


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(src: str, dst: str, extra=()) -> bool:
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(s) > t for s in (src, *extra) if os.path.exists(s))


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build_cuda(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    nvcc = _nvcc()
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s[:-3] + ".o")
        objs.append(obj)
        if force or _newer(src, obj, hdrs):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", src, "-o", obj])
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or not os.path.exists(CUDA_SO):
        _run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", CUDA_SO, *objs,
              "-Xcompiler", "-fPIC"])
    return CUDA_SO


def build_host(force: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    hdir = os.path.join(CSRC, "host")
    if not os.path.isdir(hdir):
        return HOST_SO
    srcs = sorted(os.path.join(hdir, f) for f in os.listdir(hdir) if f.endswith(".cpp"))
    hdrs = [os.path.join(hdir, f) for f in os.listdir(hdir) if f.endswith((".hpp", ".h"))]
    if not srcs:
        return HOST_SO
    if force or any(_newer(s, HOST_SO, hdrs) for s in srcs):
        _run(["g++", *CXX_FLAGS, "-shared", "-o", HOST_SO, *srcs])
    return HOST_SO


def build(force: bool = False, verbose: bool = False) -> None:
    with _lock:
        build_cuda(force, verbose)
        build_host(force)


def _preload_cudart():
    """Make sure the CUDA runtime torch uses is the one our library binds to."""
    try:
        import torch  # noqa: F401  (loads libcudart.so.12 into the process)
    except Exception:  # pragma: no cover
        pass


def cuda_lib() -> ctypes.CDLL:
    """ctypes handle on the sm_90a kernel library. Fails loudly when it is missing."""
    global _cuda_lib
    if _cuda_lib is None:
        with _lock:
            if _cuda_lib is None:
                if not os.path.exists(CUDA_SO):
                    build_cuda()
                _preload_cudart()
                _cuda_lib = ctypes.CDLL(CUDA_SO, mode=ctypes.RTLD_GLOBAL)
    return _cuda_lib


def host_lib() -> ctypes.CDLL:
    global _host_lib
    if _host_lib is None:
        with _lock:
            if _host_lib is None:
                override = os.environ.get("HCTR_HOST_LIB")     # e.g. a sanitizer build (docs/testing.md)
                if override:
                    _host_lib = ctypes.CDLL(override)
                    return _host_lib
                if not os.path.exists(HOST_SO) or os.environ.get("HCTR_REBUILD_HOST"):
                    build_host()
                _host_lib = ctypes.CDLL(HOST_SO)
    return _host_lib


def cuda_available() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # pragma: no cover
        return False


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print("built", CUDA_SO, HOST_SO)
