"""Plain restatement of skopt's θ fit for the tests: sklearn's GaussianProcessRegressor.fit with skopt's default kernel
($SK/_gpr.py:299-339), one start after another, every evaluation ``oracle.gp_oracle.lml_and_grad`` in FP64 NumPy.

θ order is sklearn's: (log amp, log ℓ_1..D, log noise).  Bounds: amp [0.01, 1000], ℓ [0.01, 100], noise [1e-5, 1e5]; sklearn's
alpha = 1e-10 sits on the diagonal with the noise.  Starts: log(1, …, 1), then ``n_restarts`` draws of
``RandomState(seed).uniform(lo, hi)``.  Each start: ``scipy.optimize.minimize(L-BFGS-B, jac=True)`` with SciPy's defaults; a
non-positive-definite θ is (+inf, 0).  The winner is np.argmin of the final −LML."""
from __future__ import annotations

import numpy as np
from scipy.linalg import LinAlgError
from scipy.optimize import minimize

from oracle import gp_oracle as O

ALPHA = 1e-10


def log_bounds(D):
    return np.log(np.array([(0.01, 1000.0)] + [(0.01, 100.0)] * D + [(1e-5, 1e5)]))


def objective(X, y, t, kind="matern52"):
    """(−LML, −gradient) in sklearn's order at θ = t."""
    amp, ls, noise = np.exp(t[0]), np.exp(t[1:-1]), np.exp(t[-1])
    try:
        lml, g = O.lml_and_grad(X, y, kind=kind, length_scale=ls if len(ls) > 1 else ls[0], amplitude=amp, noise=noise + ALPHA)
    except (LinAlgError, np.linalg.LinAlgError):
        return np.inf, np.zeros(len(t))
    # lml_and_grad: (log amp, log(noise + alpha), log ℓ…); sklearn differentiates with respect to log noise alone
    return -lml, -np.concatenate([[g[0]], g[2:], [g[1] * noise / (noise + ALPHA)]])


def skopt_theta_fit(X, y, *, seed, n_restarts=2, kind="matern52", maxiter=None):
    X = np.asarray(X, dtype=np.float64)
    D = X.shape[1]
    b = log_bounds(D)
    rng = np.random.RandomState(seed)
    x0s = [np.zeros(D + 2)] + [rng.uniform(b[:, 0], b[:, 1]) for _ in range(n_restarts)]
    runs = []
    for x0 in x0s:
        r = minimize(lambda t: objective(X, y, t, kind), x0, method="L-BFGS-B", jac=True, bounds=b,
                     options={} if maxiter is None else dict(maxiter=maxiter))
        runs.append(dict(theta0=x0, theta=r.x, neg_lml=float(r.fun), nit=int(r.nit), nfev=int(r.nfev), status=int(r.status)))
    w = int(np.argmin([r["neg_lml"] for r in runs]))
    return dict(theta=runs[w]["theta"], lml=-runs[w]["neg_lml"], winner=w, starts=runs)


def golden_cases(path):
    z = np.load(path)
    out = {}
    for name in z["names"]:
        out[str(name)] = {f: z[f"{name}__{f}"] for f in ("X", "y", "random_state", "seed", "theta0", "theta", "neg_lml", "kernel_theta", "lml")}
    return out
