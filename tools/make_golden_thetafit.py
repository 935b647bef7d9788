"""Golden θ fits from the REAL scikit-learn GaussianProcessRegressor as skopt's default GP configures it -> tests/golden/thetafit_cases.npz.

Kernel ConstantKernel(1.0, (0.01, 1000)) * Matern(ν = 2.5, ℓ = ones(D), bounds (0.01, 100)) + WhiteKernel() (noise 1, bounds
(1e-5, 1e5)), alpha = 1e-10, normalize_y = True, n_restarts_optimizer = 2, random_state = the seed skopt's Optimizer would hand
cook_estimator.  ``_constrained_optimization`` is wrapped to record each start's initial θ, final θ and −LML; the fitted
``kernel_.theta`` and ``log_marginal_likelihood_value_`` are recorded too.  θ order is sklearn's: (log amp, log ℓ_1..D, log noise).
scikit-learn is needed here only.  Run:  python tools/make_golden_thetafit.py"""
import os
import sys

import numpy as np
import sklearn
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubeflow_b200.thetafit import estimator_seed  # noqa: E402


class RecordingGPR(GaussianProcessRegressor):
    def _constrained_optimization(self, obj_func, initial_theta, bounds):
        theta, fmin = super()._constrained_optimization(obj_func, initial_theta, bounds)
        self.record_.append((np.array(initial_theta, dtype=np.float64), np.array(theta, dtype=np.float64), float(fmin)))
        return theta, fmin


def cases():
    r = np.random.default_rng(2024)
    out = []
    for N, D in ((20, 1), (60, 3), (150, 6)):          # smooth target, near-noiseless
        X = r.random((N, D))
        out.append((f"smooth_n{N}_d{D}", X, np.sin(4 * X @ np.linspace(1, 0.5, D)) + 1e-6 * r.standard_normal(N), 11 + N))
    X = r.random((60, 3))
    out.append(("noisy_n60_d3", X, np.sin(3 * X.sum(1)) + 0.3 * r.standard_normal(60), 5))
    X = r.random((60, 3))                              # dimension 2 is irrelevant: its ℓ runs to the upper bound
    out.append(("irrelevant_n60_d3", X, np.cos(3 * X[:, 0]) + X[:, 1] ** 2 + 1e-3 * r.standard_normal(60), 7))
    X = r.random((20, 3))
    out.append(("smooth_n20_d3", X, (X ** 2).sum(1), 3))
    return out


def main():
    out = {}
    for name, X, y, random_state in cases():
        D = X.shape[1]
        seed = estimator_seed(random_state)
        kernel = ConstantKernel(1.0, (0.01, 1000.0)) * Matern(length_scale=np.ones(D), length_scale_bounds=[(0.01, 100)] * D, nu=2.5) + WhiteKernel()
        gpr = RecordingGPR(kernel=kernel, alpha=1e-10, normalize_y=True, n_restarts_optimizer=2, random_state=seed)
        gpr.record_ = []
        gpr.fit(X, y)
        rec = gpr.record_
        out[name] = dict(X=X, y=y, random_state=random_state, seed=seed, theta0=np.stack([a for a, _, _ in rec]),
                         theta=np.stack([b for _, b, _ in rec]), neg_lml=np.array([c for _, _, c in rec]),
                         kernel_theta=gpr.kernel_.theta, lml=gpr.log_marginal_likelihood_value_)
        print(f"{name}: winner {int(np.argmin(out[name]['neg_lml']))} lml {gpr.log_marginal_likelihood_value_:.6f} "
              f"θ {np.round(gpr.kernel_.theta, 4)}")
    path = os.path.join(ROOT, "tests", "golden", "thetafit_cases.npz")
    np.savez_compressed(path, sklearn_version=sklearn.__version__, names=np.array(sorted(out)),
                        **{f"{k}__{f}": v[f] for k, v in out.items() for f in v})
    print(path)


if __name__ == "__main__":
    main()
