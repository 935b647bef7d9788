"""CPU: the CMA-ES termination test in the built libkbo.so (cuobjdump -sass; no GPU needed).  Its no-effect criteria are
exact FP64 equality tests, so each product and sum must round on its own (DMUL / DADD, never a contracted DFMA), and √C_ii
and max(d)/min(d) come from integer routines rather than the DFMA Newton sequences of FP64 sqrt and division.  Everything
stays in registers and shared memory (no local memory)."""
import shutil

import pytest

from kubeflow_b200 import build
from tests.test_sass_forest import _ops


@pytest.fixture(scope="module")
def built():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()


def test_stop_kernel_rounds_every_step_and_keeps_no_local_memory(built):
    (ops,) = _ops(r"cma_stop_kernel").values()
    assert any(o.startswith("DMUL") for o in ops) and any(o.startswith("DADD") for o in ops)
    assert not any(o.startswith("DFMA") for o in ops)
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
