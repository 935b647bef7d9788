"""CPU: the separable CMA-ES kernels in the built libkbo.so (cuobjdump -sass; no GPU needed).  They keep everything in
registers and shared memory (no local memory) and reduce in a fixed order without atomics, so the same calls give
bit-identical states.  The termination test's no-effect criterion is an exact FP64 equality test, so, as in
cma_stop_kernel, every product and sum rounds on its own (DMUL / DADD, never a contracted DFMA)."""
import shutil

import pytest

from kubeflow_b200 import build
from tests.test_sass_forest import _ops


@pytest.fixture(scope="module")
def built():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()


@pytest.mark.parametrize("kernel", [r"sepcma_update_kernel", r"sepcma_finish_kernel", r"sepcma_should_stop_kernel"])
def test_sep_kernels_keep_no_local_memory_and_no_atomics(built, kernel):
    (ops,) = _ops(kernel).values()
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
    assert not any(o.startswith(("ATOM", "RED")) for o in ops)
    assert any(o.startswith(("DADD", "DFMA", "DMUL")) for o in ops)


def test_sep_stop_kernel_rounds_every_step(built):
    (ops,) = _ops(r"sepcma_should_stop_kernel").values()
    assert any(o.startswith("DMUL") for o in ops) and any(o.startswith("DADD") for o in ops)
    assert not any(o.startswith("DFMA") for o in ops)
