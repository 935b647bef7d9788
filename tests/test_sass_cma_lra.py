"""CPU: the learning-rate adaptation kernels in the built libkbo.so (cuobjdump -sass; no GPU needed).  They keep everything
in registers and shared memory (no local memory) and reduce in a fixed order without atomics, so the same calls give
bit-identical states.  The kernels the plain path runs are untouched: their SASS is the parent commit's (a per-function
diff when the adaptation was added)."""
import shutil

import pytest

from kubeflow_b200 import build
from tests.test_sass_forest import _ops


@pytest.fixture(scope="module")
def built():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()


@pytest.mark.parametrize("kernel", [r"cma_lra_prep_kernel", r"cma_lra_kernel", r"cma_lra_finish_kernel"])
def test_lra_kernels_keep_no_local_memory_and_no_atomics(built, kernel):
    (ops,) = _ops(kernel + r"P").values()
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
    assert not any(o.startswith(("ATOM", "RED")) for o in ops)
    assert any(o.startswith(("DADD", "DFMA", "DMUL")) for o in ops)
