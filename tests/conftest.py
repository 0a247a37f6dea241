import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: minutes per test (the reference's test_bkz over the forwarded GSO): run with "
                                       "B200_TEST_SLOW=1")
    config.addinivalue_line("markers", "multigpu: needs two GPUs in one box (gpurun --gpus 2)")


def _visible_gpus():
    try:
        import torch
        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


def pytest_collection_modifyitems(config, items):
    """The slow tests are DESELECTED (and reported as such) unless B200_TEST_SLOW=1; the two-GPU ones are skipped on a
    machine with fewer than two devices."""
    slow_on = bool(os.environ.get("B200_TEST_SLOW"))
    ngpu = None
    keep, drop = [], []
    for it in items:
        if it.get_closest_marker("slow") and not slow_on:
            drop.append(it)
            continue
        if it.get_closest_marker("multigpu"):
            if ngpu is None:
                ngpu = _visible_gpus()
            if ngpu < 2:
                it.add_marker(pytest.mark.skip(reason="needs two GPUs in one machine"))
        keep.append(it)
    if drop:
        config.hook.pytest_deselected(items=drop)
        items[:] = keep


@pytest.fixture(scope="session", autouse=True)
def _build_everything():
    """Build the oracle (C restatement) and, where it is stale, the CUDA extension (nvcc cross-compiles on CPU)."""
    from oracle import build as ob
    ob.build_oracle()
    import shutil
    if shutil.which("nvcc"):
        from fplll_b200 import build as pb
        pb.build_all()
    yield
