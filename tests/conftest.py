import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "dist: multi-process test (gloo on CPU, nccl on GPU)")


def pytest_collection_modifyitems(config, items):
    import torch
    # emulated-rank tests run rank threads that rendezvous: a bug must fail fast instead of hanging the
    # (metered) GPU box until the outer timeout
    for it in items:
        if "test_emu_ranks" in it.nodeid or "test_metrics_dist" in it.nodeid:
            it.add_marker(pytest.mark.timeout(180))
    # HCTR_GPU_TESTS_ON_CPU=1: development aid -- run the bodies of the gpu-marked tests on the CPU
    # reference paths (those that do not address a cuda device explicitly) to find CPU-path regressions
    if torch.cuda.is_available() or os.environ.get("HCTR_GPU_TESTS_ON_CPU") == "1":
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)

