import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


# Collection order of the GPU suites: kernel-level pins first (tracker, EKF kernels), then the pipeline suites, then the
# widened rows -- a failing workload-level assertion must never hide the kernel parity evidence behind `-x`.
_ORDER = ["test_gpu_tracker", "test_gpu_ekf", "test_gpu_brief", "test_gpu_estimator", "test_gpu_widen", "test_gpu_bench_workload"]


def pytest_collection_modifyitems(session, config, items):
    def key(it):
        name = os.path.basename(str(it.fspath))
        for i, pre in enumerate(_ORDER):
            if name.startswith(pre):
                return i
        return len(_ORDER) if name.startswith("test_gpu") else -1

    items.sort(key=key)  # stable: the order inside a module is kept


@pytest.fixture(scope="session")
def ctx():
    """CUDA context through the C ABI.  No skip-on-missing: a GPU test without a GPU or without
    the built library must fail loudly (there is no CPU fallback to fall back to)."""
    from xivo_b200 import Context

    c = Context(0)
    yield c
    c.close()
