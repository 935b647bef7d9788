"""CPU: the GBRT kernels in the built libkbo.so (cuobjdump -sass; no GPU needed).  No kernel the GBRT path launches touches
local memory, its own or the tree_*_kernel it shares with the forests (kbo_tree.cuh); the staged sweep reads the model and the
candidate tile from shared memory; the predict instances of the sweep — the chain sums alone — hold no DFMA, so every stage's
fl(0.1·v) is added with a plain DADD as sklearn adds it."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build


def _ops(kernel_pattern):
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
        elif name and re.search(kernel_pattern, name):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                out.setdefault(name, []).append(m.group(1))
    return out


@pytest.fixture(scope="module")
def built():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()


def test_no_gbrt_path_kernel_uses_local_memory(built):
    kernels = _ops(r"gbrt_|tree_(check|keys|reduce)_kernel")
    assert len(kernels) == 9, sorted(kernels)      # init, fit, 4 sweep instances; check, keys, reduce
    for name, ops in kernels.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name


def test_sweep_instances(built):
    kernels = _ops(r"gbrt_sweep_kernel")
    assert len(kernels) == 4, sorted(kernels)
    for name, ops in kernels.items():
        assert any(o.startswith("DADD") for o in ops), name
        if "ILb1E" in name:                                   # the staged instances
            assert any(o.startswith("LDS") for o in ops), name
        if name.endswith("Lb0EEv13GbrtSweepArgs"):           # predict: the sums alone
            assert not any(o.startswith("DFMA") for o in ops), name

