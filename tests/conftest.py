import os
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def _gpu_ok():
    try:
        import librosa_b200 as lb

        lb.default_context()
        return True
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU must fail loudly, not skip: the product has no CPU fallback.
    return


@pytest.fixture(scope="session")
def golden():
    out = {}
    for name in ("hotpath_v1.npz", "features_v1.npz"):
        with np.load(os.path.join(ROOT, "tests", "golden", name)) as z:
            out.update({k: z[k] for k in z.files})
    return out


@pytest.fixture(scope="session")
def oracle():
    from oracle import ref_np

    return ref_np


def case_input(case):
    import signals

    sr = case["kw"].get("sr", 22050)
    return signals.make(case["mix"], case["shape"], seed=len(case["name"]), sr=sr)
