"""CPU: the built libkbo.so really contains the sm_90a instructions DESIGN.md claims, kernel by kernel (cuobjdump -sass; no GPU needed).
A refactor that silently falls back to mma.sync / plain loads, or drops the TMA multicast path, fails here."""
import re
import shutil
import subprocess

import pytest

from kubeflow_b200 import _lib, build


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    build.build()
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
            if m:
                kernels[name].append(m.group(1))
    return kernels


def _ops(sass, needle):
    hits = [ops for name, ops in sass.items() if needle in name]
    assert hits, f"no kernel named *{needle}* in libkbo.so"
    return [o for ops in hits for o in ops]


def test_ranking_kernel_is_wgmma_with_tma(sass):
    ops = _ops(sass, "tc_rank_kernel")
    assert any(o.startswith("HGMMA.64x256x16.F32") for o in ops)         # wgmma.mma_async m64n256k16, fp32 accumulate
    assert any(o.startswith("UTMALDG") for o in ops)                      # cp.async.bulk.tensor
    assert any(o.startswith("SYNCS.PHASECHK") for o in ops)               # mbarrier.try_wait


def test_kstar_kernel_is_wgmma_plus_two_mufu_per_pair(sass):
    ops = _ops(sass, "tc_kstar_kernelILi1")
    assert any(o.startswith("HGMMA") for o in ops) and any(o.startswith("UTMALDG") for o in ops)
    assert ops.count("MUFU.SQRT") >= 64 and ops.count("MUFU.EX2") >= 64 and "MUFU.RSQ" not in ops


def test_three_product_kernel_uses_tma_multicast(sass):
    ops = _ops(sass, "tc_variance_kernel")
    assert any(o.startswith("HGMMA") for o in ops) and any("MULTICAST" in o for o in ops if o.startswith("UTMALDG"))


def test_fp64_gemm_runs_on_the_fp64_tensor_cores(sass):
    for needle in ("dgemm64_kernelILb1ELi0", "dgemm64_kernelILb0ELi0"):
        ops = _ops(sass, needle)
        assert ops.count("DMMA.8x8x4") >= 64, needle


def test_diagonal_block_kernel_has_no_local_memory_and_one_seed_per_column(sass):
    ops = _ops(sass, "potf2_inv_kernel")
    assert not any(o.startswith(("LDL", "STL")) for o in ops)             # the 16-column register tile stays in registers
    assert ops.count("MUFU.RSQ64H") == 16                                  # hardware seed of 1/sqrt, once per column step
