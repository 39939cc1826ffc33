import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.dirname(os.path.abspath(__file__))
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

P = 0xFFFFFFFF00000001


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _splitmix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = x
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def synth(seed, shape, canonical=True):
    """Counter-based synthetic field elements (SURVEY.md section 8d): splitmix64(seed, idx)."""
    n = int(np.prod(shape))
    with np.errstate(over="ignore"):
        idx = np.arange(n, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x1000000000)
        v = _splitmix64(idx)
        if canonical:
            v = np.where(v >= np.uint64(P), v - np.uint64(P), v)
    return v.reshape(shape)


EDGE = [0, 1, P - 1, P - 2, 2**32 - 1, 2**32, 2**63, P - 2**32, 2**64 - 1, P, P + 1, 2**64 - 2**32]


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib

    oracle_lib.lib()
    return oracle_lib
