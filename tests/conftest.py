import os
import sys

import numpy as np
import pytest

os.environ.setdefault("FIDGET_B200_ENV_LIVE", "1")   # tests flip tuning knobs between calls: re-read them every time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MODELS = os.path.join(ROOT, "models")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")


def model_text(name):
    with open(os.path.join(MODELS, name)) as f:
        return f.read()


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (test infrastructure)."""
    from oracle import oracle as o
    o.lib()
    return o


@pytest.fixture(scope="session")
def cuda():
    """A CudaContext on device 0.  gpu-marked tests FAIL (not skip) without a device."""
    import fidget_b200 as fb
    return fb.CudaContext(0)


@pytest.fixture(scope="session")
def models():
    return model_text


def same_f32(a, b):
    """Bitwise equality of float arrays, treating every NaN as equal."""
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb]))
