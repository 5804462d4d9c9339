import os
import sys

# the float64 oracle does many small matmuls: a 128-thread BLAS pool on the GPU box makes them crawl
for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(_v, "8")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible, e.g. a plain `pytest tests/` here."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session", autouse=True)
def _limit_blas_threads():
    try:
        from threadpoolctl import threadpool_limits
        with threadpool_limits(limits=8):
            yield
    except ImportError:  # pragma: no cover
        yield
