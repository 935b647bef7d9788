"""How far is an fp32 acquisition value off when y is not centred?  (CPU only; not collected by pytest.)

The sweep's fp32 kernels once formed μ = y_mean + y_std·μ_n and imp = y_opt − ξ − μ in fp32, so μ was rounded at the scale of
y_mean.  This emulates that arithmetic in NumPy float32 on the exact oracle posterior (N = 1000, M = 60 000, D = 6, Matérn-5/2,
EI, y = c + s·y₀) and compares it, and the normalised frame the kernels use now (c_n = (y_opt − ξ − y_mean)/y_std in FP64 as
an fp32 hi/lo pair, imp_n = c_n − μ_n, EI = y_std·(imp_n·Φ + σ_n·φ)), with the FP64 values.

    python tests/studies/acq_f32_offset_study.py
"""
import os
import sys

import numpy as np
from scipy.special import ndtr

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import gp_oracle as O  # noqa: E402

f32 = np.float32


def ei_f32(z_imp, sd):
    z = z_imp / sd
    return z_imp * f32(ndtr(z)) + sd * f32(np.exp(-0.5 * z.astype(np.float64) ** 2) / np.sqrt(2 * np.pi))


def main():
    N, M, D = 1000, 60_000, 6
    X, y0, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    print(f"N={N} M={M} D={D} Matern-5/2 EI\n{'c':>9} {'s':>4} {'max EI':>8} {'raw frame':>10} {'normalised':>11}")
    for c, s in [(0.0, 1.0), (1e3, 1.0), (2e4, 5.0), (-1e5, 2.0)]:
        y = c + s * y0
        fit = O.gp_fit(X, y, kind="matern52", length_scale=th["length_scale"], amplitude=1.0, noise=th["noise"])
        mu, sd = O.gp_predict(fit, Xc)
        y_opt, ym, ys, xi = float(y.min()), fit["y_mean"], fit["y_std"], th["xi"]
        ref = O.acquisition(mu, sd, y_opt, "ei", xi)
        mun = ((mu - ym) / ys).astype(f32)                      # what the kernels read: fp32 μ_n, σ²_n
        varn = ((sd / ys) ** 2).astype(f32)
        sdn = np.sqrt(varn)
        # before: raw frame in fp32
        mu32 = f32(ys) * mun + f32(ym)
        imp32 = f32(y_opt) - f32(xi) - mu32
        old = ei_f32(imp32, sdn * f32(ys)).astype(np.float64)
        # now: normalised frame
        cn = (y_opt - xi - ym) / ys
        chi = f32(cn)
        clo = f32(cn - float(chi))
        new = ys * ei_f32((chi - mun) + clo, sdn).astype(np.float64)
        print(f"{c:>9g} {s:>4g} {ref.max():8.3f} {np.abs(old - ref).max():10.1e} {np.abs(new - ref).max():11.1e}")


if __name__ == "__main__":
    main()
