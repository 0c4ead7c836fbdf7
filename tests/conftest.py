import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def engine():
    """One CUDA engine for the whole GPU test session (fails loudly if the .so is missing)."""
    from lungmask_b200 import _native
    eng = _native.Engine(device=0, batch_capacity=4)
    yield eng
    eng.close()


@pytest.fixture(scope="session")
def ct_slice():
    """The real CT slice of the reference's tests/testdata/0.dcm (pixel data only), see tests/golden/README.md."""
    import numpy as np
    p = os.path.join(ROOT, "tests", "golden", "ct_slice_512.npz")
    return np.load(p)["slice"]
