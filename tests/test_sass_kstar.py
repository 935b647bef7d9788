"""CPU: both instantiations of the tensor-core K* kernel (RBF and Matérn) keep everything in registers and shared memory
(cuobjdump -sass of the built libkbo.so; no GPU needed).  A spill in its epilogue would put local-memory traffic on every tile."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build


def _kstar_kernels():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "tc_kstar_kernel" in m.group(1) else None
            if name:
                kernels[name] = []
        elif name:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                kernels[name].append(m.group(1))
    return kernels


def test_kstar_kernel_has_no_local_memory_in_either_instantiation():
    kernels = _kstar_kernels()
    assert any("ILi0" in n for n in kernels) and any("ILi1" in n for n in kernels), sorted(kernels)
    for name, ops in kernels.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("LDS.128") for o in ops), name     # the (|x̂|², α) pairs come from shared memory
        assert not any(o.startswith("LD.E") for o in ops), name    # ... through LDS, not generic loads
