"""CPU: the forest kernels in the built libkbo.so (cuobjdump -sass; no GPU needed).  The sweep reads the staged tree nodes
and leaf records from shared memory (LDS) and keeps everything else in registers (no local memory in its walk); the leaf
records' v² + impurity and the sweep's accumulation are plain DMUL / DADD (__dmul_rn / __dadd_rn), never a contracted DFMA,
so the device sums round exactly like the NumPy restatement's."""
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


def test_sweep_kernels_read_nodes_from_shared_memory_without_local_memory(built):
    kernels = _ops(r"forest_sweep_kernel")
    assert len(kernels) == 4, sorted(kernels)
    for name, ops in kernels.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("DADD") for o in ops), name
        if "Lb1E" in name:                                   # the staged instances
            assert any(o.startswith("LDS.64") for o in ops), name   # nodes
            assert any(o.startswith("LDS.128") for o in ops), name  # leaf records


SWEEP_STATIC_SMEM = 768      # TreeArgmax::write's kbo_best sp[3][8]; tests/test_gpu_tree_scale.py derives its staging band from it


def _shared_bytes(kernel_pattern):
    txt = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"\bSHARED:(\d+)", line)
        if m and name and re.search(kernel_pattern, name):
            out[name] = int(m.group(1))
    return out


def test_sweep_kernels_static_shared_memory_is_the_size_the_staging_band_assumes(built):
    """The staged sweep may opt in to (per-block limit − static) bytes of dynamic shared memory for a tree: the band of tree sizes
    where that matters is derived from this static size.  sm_90 code objects count the 1 KiB the system reserves per block in
    every kernel's shared size: a kernel without shared variables shows exactly that."""
    (reserved,) = _shared_bytes(r"forest_bootstrap_kernel").values()
    assert reserved == 1024
    sweeps = _shared_bytes(r"forest_sweep_kernel")
    assert len(sweeps) == 4, sorted(sweeps)
    for name, b in sweeps.items():
        assert b - reserved == SWEEP_STATIC_SMEM, f"{name}: {b - reserved} static bytes; re-derive the band in test_gpu_tree_scale.py"


def test_leaf_records_are_formed_without_fma(built):
    (ops,) = _ops(r"forest_pack_kernel").values()
    assert any(o.startswith("DMUL") for o in ops) and any(o.startswith("DADD") for o in ops)
    assert not any(o.startswith("DFMA") for o in ops)
