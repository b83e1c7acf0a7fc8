import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")
    config.addinivalue_line("markers", "slow: long-running CPU test")


def _usable_cores():
    import os
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    try:  # cgroup v2 CPU quota
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(int(q) / int(per))))
    except Exception:
        pass
    return n


try:
    import torch
    # the fp32 oracle (CPU torch) is fastest with a moderate thread count; many-core boxes oversubscribe badly
    torch.set_num_threads(max(1, min(16, _usable_cores())))
except Exception:
    pass
