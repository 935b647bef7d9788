"""How well do the calibration rows predict the ranking pass's error on the rest of the grid?  (DESIGN.md §1, kbo_set_tc_fast)

CPU emulation of the one-product pass — K* and W = L⁻¹ rounded to fp16 (W scaled as split_w_kernel does), exact accumulation —
against the fp64 Σv², for a few fits of the workload of record: max |dσ²| over the first 18 944 candidates (what calib_kernel
sees: one wave of sm_count CTAs × 128 rows) versus the maximum over the whole grid.  Uses the oracle, hence lives under
tests/.  Output of the run recorded in DESIGN.md (2 min on 8 cores):

    N=2048 D=32 matern52: calibration rows 1.024e-03, all 160000 rows 1.141e-03, ratio 1.11
    N=2048 D=8  rbf:      calibration rows 4.052e-02, all 160000 rows 4.056e-02, ratio 1.00
    N=1024 D=5  rbf:      calibration rows 2.862e-02, all 160000 rows 2.862e-02, ratio 1.00
    N=3000 D=16 matern52: calibration rows 1.848e-03, all 120000 rows 1.912e-03, ratio 1.03
"""
import numpy as np

from oracle import gp_oracle as O


def study(N, M, D, kind):
    X, y, _ = O.synthetic(N, 1, D)
    th = O.theta_of_record(D)
    fit = O.gp_fit(X, y, kind=kind, length_scale=th["length_scale"], amplitude=1.0, noise=th["noise"])
    W = np.linalg.inv(fit["L"])
    sc = 2.0 ** (14 - np.ceil(np.log2(np.abs(W).max())))
    Wh = ((W * sc).astype(np.float16).astype(np.float64) / sc).T.copy()
    Wt = W.T.copy()
    rng = np.random.default_rng(4321)
    ds = []
    for s in range(0, M, 8192):
        Xc = rng.random((min(8192, M - s), D))
        Ks = O.kernel_matrix(Xc, fit["X"], fit["length_scale"], kind, 1.0)
        Kh = Ks.astype(np.float16).astype(np.float64)
        v, v1 = Ks @ Wt, Kh @ Wh
        ds.append((v1 * v1).sum(1) - (v * v).sum(1))
    d = np.abs(np.concatenate(ds))
    print(f"N={N} D={D} {kind}: calibration rows {d[:18944].max():.3e}, all {M} rows {d.max():.3e}, ratio {d.max() / d[:18944].max():.2f}")


if __name__ == "__main__":
    study(2048, 160000, 32, "matern52")
    study(2048, 160000, 8, "rbf")
    study(1024, 160000, 5, "rbf")
    study(3000, 120000, 16, "matern52")
