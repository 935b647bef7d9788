"""CPU: the CMA-ES with Margin kernels in the built libkbo.so (cuobjdump -sass; no GPU needed).  The margin kernel keeps
everything in registers (no local memory), and both kernels form levels and thresholds with DMUL / DADD as NumPy does,
so a sample encodes to the same level as the oracle's.  The margin-free kernels are untouched: their SASS is the parent
commit's (compared with tools/sass_summary.py and a per-instruction diff when the margin was added)."""
import shutil

import pytest

from kubeflow_b200 import build
from tests.test_sass_forest import _ops


@pytest.fixture(scope="module")
def built():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()


@pytest.mark.parametrize("kernel", [r"cma_margin_kernel", r"cma_x_margin_kernel"])
def test_margin_kernels_keep_no_local_memory(built, kernel):
    (ops,) = _ops(kernel).values()
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
    assert any(o.startswith("DMUL") for o in ops) and any(o.startswith("DADD") for o in ops)
