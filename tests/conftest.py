import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def golden_cases():
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, "gp_*.npz")))


def load_golden(path):
    z = np.load(path, allow_pickle=False)
    d = {k: z[k] for k in z.files}
    for k in ("kind", "acq_kind"):
        d[k] = str(d[k])
    for k in ("amplitude", "noise", "xi", "kappa", "y_mean", "y_std", "lml"):
        d[k] = float(d[k])
    d["index"] = int(d["index"])
    d["name"] = os.path.basename(path)[3:-4]
    return d


@pytest.fixture(params=golden_cases(), ids=lambda p: os.path.basename(p)[3:-4])
def golden(request):
    return load_golden(request.param)
