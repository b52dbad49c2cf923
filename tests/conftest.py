import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100 box)")


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


@pytest.fixture(scope="session")
def n_gpus():
    return _n_gpus()


# `-m gpu -x` order: the watchdogged smoke case, then the single-GPU product-path parity tests, then the full-size baseline
# configurations, then the multi-GPU suites (which skip on a smaller box) -- a failure late in the list cannot hide the
# results of the tests every box can run
GPU_FILE_ORDER = {"test_gpu_00_smoke.py": 1, "test_gpu_parity.py": 2, "test_gpu_baseline_configs.py": 3, "test_gpu_multi.py": 4,
                  "test_gpu_zz_reference_golden.py": 5}


def pytest_collection_modifyitems(config, items):
    items.sort(key=lambda it: GPU_FILE_ORDER.get(os.path.basename(str(it.fspath)), 0))   # stable: order inside a file is kept
    # `-m gpu` on a box without a GPU must fail loudly rather than skip silently; plain runs
    # (no -m) on a CPU box skip GPU tests.
    if _n_gpus() == 0 and "gpu" not in (config.getoption("-m") or ""):
        skip = pytest.mark.skip(reason="no CUDA device")
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)
