import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not errored) on a host without CUDA or without the built library, so that a plain
    `pytest tests` on a CPU box still shows the CPU suite's verdict."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    have_lib = os.path.exists(os.path.join(ROOT, "polara_b200", "libpolara_b200.so"))
    if have_gpu and have_lib:
        return
    why = "no CUDA device" if not have_gpu else "libpolara_b200.so is not built"
    skip = pytest.mark.skip(reason="gpu test: " + why)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def golden():
    return load_golden
