"""CPU: the ENAS kernels in the built libkbo.so, as the design describes them (cuobjdump -sass; no GPU needed).  The train
kernel keeps its state in registers and shared memory (no LDL / STL), sums with fixed-order warp shuffles (SHFL.BFLY) and
never uses atomics, which is what makes its results bit-reproducible; it is one CTA, so it has no cluster or DSMEM traffic."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build


def _ops(kernel: str) -> list:
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    ops, name = [], None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
        elif name and kernel in name:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                ops.append(m.group(1))
    assert ops, f"{kernel} not found in the library"
    return ops


@pytest.mark.parametrize("kernel", ["enas_train_kernel", "enas_sample_kernel"])
def test_enas_kernels_have_no_local_memory_and_no_atomics(kernel):
    ops = _ops(kernel)
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
    assert not any(o.startswith(("ATOM", "RED", "ATOMS")) for o in ops)
    assert any(o.startswith("SHFL.BFLY") for o in ops) and any(o.startswith("BAR.SYNC") for o in ops)
    assert not any(o.startswith(("UCGABAR", "CGAERRBAR")) for o in ops)     # no cluster barrier: one CTA per chain
