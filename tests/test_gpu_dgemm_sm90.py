"""GPU: the fit's FP64 GEMM (dgemm_sm90_kernel, m16n8k8 DMMA) against a NumPy FP64 product on sizes that are not multiples of
the 128×64×16 tile, for every K-range mode, both operand layouts, lower-tile skipping and the alpha = ±1, beta = 1 preload path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

KM_FULL, KM_UPTO_N, KM_FROM_N, KM_UPTO_M, KM_FROM_M = range(5)
TS_NONE, TS_LOWER = 0, 1
BM, BN, BK = 128, 64, 16


def _expected(A, B, C0, transb, alpha, beta, kmode, kbegin, tileskip):
    """The kernel's contract, tile by tile: row tile m0, column tile n0 sum over k in [kb, ke) with kb, ke clipped as kmode says."""
    M, N, K = C0.shape[0], C0.shape[1], A.shape[1]
    Bk = B.T if transb else B   # K × N
    out = C0.copy()
    for m0 in range(0, M, BM):
        for n0 in range(0, N, BN):
            if tileskip == TS_LOWER and n0 > m0 + BM - 1:
                continue
            kb, ke = kbegin, K
            if kmode == KM_UPTO_N:
                ke = min(K, n0 + BN)
            if kmode == KM_FROM_N:
                kb = max(kbegin, n0)
            if kmode == KM_UPTO_M:
                ke = min(K, m0 + BM)
            if kmode == KM_FROM_M:
                kb = max(kbegin, m0)
            kb = max(kbegin, kb & ~(BK - 1))
            rm, rn = slice(m0, min(M, m0 + BM)), slice(n0, min(N, n0 + BN))
            prod = A[rm, kb:ke] @ Bk[kb:ke, rn] if ke > kb else 0.0
            out[rm, rn] = alpha * prod + beta * C0[rm, rn]
    return out


CASES = [
    # (M, N, K, transb, alpha, beta, kmode, kbegin, tileskip)
    (301, 197, 259, True, -1.0, 1.0, KM_FULL, 0, TS_NONE),
    (301, 301, 259, True, -1.0, 1.0, KM_FULL, 0, TS_LOWER),
    (257, 129, 77, True, 1.0, 1.0, KM_FULL, 0, TS_NONE),
    (300, 200, 190, True, 1.0, 0.0, KM_UPTO_N, 0, TS_NONE),
    (173, 250, 333, False, 1.0, 0.0, KM_FROM_N, 0, TS_NONE),
    (250, 173, 250, False, -1.0, 0.0, KM_UPTO_M, 0, TS_NONE),
    (250, 173, 300, True, 1.0, 0.0, KM_FROM_M, 0, TS_NONE),
    (199, 131, 211, False, 1.0, 0.0, KM_FULL, 37, TS_NONE),
    (199, 131, 211, True, 0.5, 2.0, KM_FULL, 5, TS_NONE),
    (17, 9, 3, False, -1.0, 1.0, KM_FULL, 0, TS_NONE),
]


@pytest.mark.parametrize("M,N,K,transb,alpha,beta,kmode,kbegin,tileskip", CASES)
def test_dgemm_sm90_matches_host_product(M, N, K, transb, alpha, beta, kmode, kbegin, tileskip):
    from kubeflow_b200 import _lib
    from kubeflow_b200.gp import GPEngine
    rng = np.random.default_rng(M * 7919 + N * 31 + K)
    lda, ldb, ldc = K + 3, (K if transb else N) + 5, N + 2   # odd leading dimensions: no alignment beyond 8 bytes
    A = rng.standard_normal((M, lda))
    B = rng.standard_normal((N, ldb) if transb else (K, ldb))
    C0 = rng.standard_normal((M, ldc))
    dev = torch.device("cuda", 0)
    Ad, Bd, Cd = (torch.tensor(x, device=dev) for x in (A, B, C0))
    eng = GPEngine(0, kernel="rbf")
    try:
        s = torch.cuda.current_stream(dev)
        rc = eng.lib.kbo_debug_dgemm_sm90(eng._h, int(transb), M, N, K, Ad.data_ptr(), lda, Bd.data_ptr(), ldb, Cd.data_ptr(), ldc, alpha, beta,
                                          kmode, kbegin, tileskip, s.cuda_stream)
        _lib.check(eng.lib, eng._h, rc)
        torch.cuda.synchronize()
    finally:
        eng.close()
    got = Cd.cpu().numpy()
    Bv = B[:, :K] if transb else B[:, :N]
    want = _expected(A[:, :K], Bv, C0[:, :N], transb, alpha, beta, kmode, kbegin, tileskip)
    # FP64 rounding of a K-term dot product, relative to the magnitudes summed
    scale = np.abs(A[:, :K]) @ np.abs(Bv.T if transb else Bv) * abs(alpha) + abs(beta) * np.abs(C0[:, :N])
    err = np.abs(got[:, :N] - want)
    assert np.all(err <= 4 * (K + 2) * np.finfo(np.float64).eps * (scale + 1e-300)), float(np.max(err / (scale + 1e-300)))
    assert np.array_equal(got[:, N:], C0[:, N:])   # the columns past N of each row are untouched
