import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def batch_of(g):
    return {k: g[k] for k in ("obs", "act", "rew", "last_obs", "ep_offsets", "ep_done")}


def rel_err(x, ref):
    """norm-wise error: max|x-ref| / max|ref|  (SURVEY.md Appendix D: the parity bar is 1e-5 of max|ref|)."""
    x, ref = np.asarray(x, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    return float(np.max(np.abs(x - ref)) / max(np.max(np.abs(ref)), 1e-30))


@pytest.fixture(scope="session")
def golden():
    return load_golden
