"""CPU: the multivariate TPE score kernel in the built libkbo.so evaluates its exponentials on the MUFU pipe (ex2.approx →
MUFU.EX2) and keeps its register tile, its integer-parameter path and its bound in registers and shared memory
(cuobjdump -sass; no GPU needed).  A local-memory access would sit inside the loop over candidate × component pairs."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build


def test_mvtpe_score_kernel_uses_mufu_ex2_and_no_local_memory():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    ops, name = [], None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
        elif name and "mvtpe_score_kernel" in name:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                ops.append(m.group(1))
    assert ops, "mvtpe_score_kernel not found in the library"
    assert any(o.startswith("MUFU.EX2") for o in ops)
    assert not any(o.startswith(("LDL", "STL")) for o in ops)
    assert any(o.startswith("LDS.128") for o in ops)              # candidate and component slabs read as float4 / int4
