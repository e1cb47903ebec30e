import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def cuda_stream():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.cuda.current_stream().cuda_stream


def usable_cores() -> int:
    """Host cores this process may really use: affinity mask capped by the cgroup CPU quota (a 128-thread
    OpenMP team on a quota of a few cores makes the CPU oracle orders of magnitude slower)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(int(q) / int(p))))
    except Exception:
        pass
    return n


def pytest_sessionstart(session):
    import torch

    torch.set_num_threads(max(1, min(16, usable_cores())))
