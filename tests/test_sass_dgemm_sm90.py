"""CPU: the fit's FP64 GEMM in the built libkbo.so (cuobjdump -sass; no GPU needed) issues Hopper's m16n8k8 DMMA, is fed by
cp.async, and keeps its accumulators and fragments in registers."""
from tests.test_sass import _ops, sass  # noqa: F401  (the module-scoped SASS fixture)


def test_fit_gemm_runs_on_the_m16n8k8_dmma_without_local_memory(sass):  # noqa: F811
    for needle in ("dgemm_sm90_kernelILb1E", "dgemm_sm90_kernelILb0E"):
        ops = _ops(sass, needle)
        assert ops.count("DMMA.16x8x8") >= 16 and "DMMA.8x8x4" not in ops, needle   # 2×4 m16n8 tiles × 2 k8 steps per warp and K-slab
        assert any(o.startswith("LDGSTS") for o in ops), needle                      # cp.async ring
        assert not any(o.startswith(("LDL", "STL")) for o in ops), needle            # accumulators and fragments stay in registers
