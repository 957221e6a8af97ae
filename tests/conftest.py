import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def record(name: str, value) -> None:
    """Append a measured parity number to gpurun_out/parity.log (kept with the round's evidence)."""
    try:
        d = os.path.join(ROOT, "gpurun_out")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "parity.log"), "a") as f:
            f.write(f"{name} {value}\n")
    except OSError:
        pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    try:   # the fp64 CPU oracle: as many torch threads as the cgroup quota allows (the GPU boxes show 128 CPUs under
        # a 16-CPU quota; 128 threads there are 8x oversubscribed and ~20x slower)
        import torch

        from bench import host_cores

        torch.set_num_threads(host_cores())
    except Exception:  # pragma: no cover
        pass


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
