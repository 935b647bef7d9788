"""CPU: the kernels of the sharded ``tpe`` / ``multivariate-tpe`` ask in the built libkbo.so (the offset draws, the shard
winner and the pick) keep everything in registers and shared memory (cuobjdump -sass; no GPU needed)."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build

KERNELS = ("tpe_draw_kernel", "tpe_pick_kernel", "mvtpe_draw_kernel", "mvtpe_pick_kernel", "tpe_shard_best_kernel")


def test_shard_kernels_use_no_local_memory():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    ops, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        hit = next((k for k in KERNELS if name and k in name), None)
        if hit:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                ops.setdefault(name, []).append(m.group(1))
    for k in KERNELS:
        found = [n for n in ops if k in n]
        assert found, f"{k} not found in the library"
    for n, o in ops.items():
        assert not any(x.startswith(("LDL", "STL")) for x in o), n
