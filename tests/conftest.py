import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


# B2_TEST_EMULATE=1 runs the gpu-marked tests on the CPU with the native seams replaced by the
# oracle-backed stand-ins of tests/cpu_emulation.py.  It exists to debug the TEST CODE in the
# GPU-less build container; it proves nothing about the kernels and is never set by the driver.
EMULATE = os.environ.get("B2_TEST_EMULATE") == "1"


def device():
    return "cpu" if EMULATE else "cuda"


@pytest.fixture(autouse=True)
def _maybe_emulate(request):
    if EMULATE and "gpu" in request.keywords:
        import cpu_emulation
        with cpu_emulation.enabled():
            yield
    else:
        yield


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available() or EMULATE:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the native libraries exist (nvcc cross-compiles without a GPU)."""
    from pyro_b200 import _build
    _build.build()


def load_npz(name):
    return dict(np.load(os.path.join(GOLDEN, name), allow_pickle=False))


def load_json(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


@pytest.fixture(autouse=True)
def _clean_state():
    import pyro_b200
    pyro_b200.clear_param_store()
    torch.set_default_dtype(torch.float32)
    yield
    pyro_b200.clear_param_store()
    from pyro_b200.poutine import runtime
    del runtime._STACK[:]
    torch.set_default_dtype(torch.float32)
