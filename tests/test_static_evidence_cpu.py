"""Static evidence that needs no GPU: the built library's SASS carries the Hopper tensor-core (wgmma) / TMA
instructions in the kernels that are supposed to use them, and no hot kernel spills beyond a small stack."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "hugectr_b200", "lib", "libhctr_cuda.so")
need = pytest.mark.skipif(not (os.path.exists(LIB) and shutil.which("cuobjdump")),
                          reason="needs the built library and cuobjdump")


@need
def test_sass_gate_wgmma_tma_present():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools_dev", "sass_evidence.py"), "--check"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok:")


@need
def test_kernel_resource_report_and_spill_gate():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools_dev", "kernel_resources.py"), "--max-stack", "512"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr
    names = r.stdout
    for k in ("gemm_tc_kernel", "gemm_mxfp8_kernel", "emb_fwd_kernel", "emb_dispatch_kernel", "allreduce_twoshot_kernel",
              "emb_bwd_reduce_update_kernel", "emb_bwd_heavy_kernel", "emb_update_kernel"):
        assert k in names, k
