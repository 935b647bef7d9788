"""Golden Hamming-kernel GP fits from the REAL scikit-learn GaussianProcessRegressor as skopt configures it for an
all-categorical space -> tests/golden/hamming_cases.npz.

skopt is not a dependency, so its HammingKernel is restated below from memory [RECALL]: ``k(x, y) = exp(−Σ_j l_j·[x_j ≠ y_j])``,
gradient ``∂k/∂log l_j = −k·l_j·[x_j ≠ y_j]``, bounds (1e-5, 1e5), ``length_scale = ones(n_dims)``.  The GP is
``ConstantKernel(1.0, (0.01, 1000)) * Hamming + WhiteKernel()``, alpha = 1e-10, normalize_y = True, n_restarts_optimizer = 2,
random_state = the seed skopt's Optimizer would hand cook_estimator.  Inputs are category codes.

Recorded per case: each start's initial θ, final θ and −LML (``_constrained_optimization`` is wrapped), the fitted
``kernel_.theta`` and LML, the LML and gradient at every start and at the fit (``log_marginal_likelihood(θ, eval_gradient=True)``),
and the posterior μ and σ at candidate codes after the WhiteKernel is zeroed, as skopt does after its fit [RECALL].
θ order is sklearn's: (log amp, log l_1..D, log noise).

Flat log-marginal likelihoods.  A one-category dimension (c = 1) never differs: its l_j has an exactly zero gradient and stays
at each start's value.  A dimension the target does not depend on has an LML that is nearly flat in l_j once l_j is small
(exp(−l_j) ≈ 1): its fitted l_j drifts towards the lower bound and where L-BFGS-B stops depends on the last bits of the
gradient.  Cases with such dimensions: one_d3_n80 (dimension 0 has c = 1), mixed_d8_n512 (dimension 0 has c = 1; dimensions
4, 5 and 7 are irrelevant), flat_d3_n40 (dimension 2 is irrelevant) and noisy_d8_n200, whose third start stops at a poor
local optimum (l_0 ≈ e^10) where the LML is nearly flat along l_4 (weight 0.2 in the target): there the oracle's final log l_4
differs from sklearn's by 1.3e-3.
scikit-learn is needed here only.  Run:  python tools/make_golden_hamming.py"""
import os
import sys

import numpy as np
import sklearn
from sklearn.gaussian_process import GaussianProcessRegressor
from sklearn.gaussian_process.kernels import (ConstantKernel, Hyperparameter, Kernel, NormalizedKernelMixin, StationaryKernelMixin,
                                              WhiteKernel)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubeflow_b200.thetafit import estimator_seed  # noqa: E402


class Hamming(StationaryKernelMixin, NormalizedKernelMixin, Kernel):
    """skopt's HammingKernel [RECALL]."""

    def __init__(self, length_scale=1.0, length_scale_bounds=(1e-5, 1e5)):
        self.length_scale = length_scale
        self.length_scale_bounds = length_scale_bounds

    @property
    def anisotropic(self):
        return np.iterable(self.length_scale) and len(self.length_scale) > 1

    @property
    def hyperparameter_length_scale(self):
        if self.anisotropic:
            return Hyperparameter("length_scale", "numeric", self.length_scale_bounds, len(self.length_scale))
        return Hyperparameter("length_scale", "numeric", self.length_scale_bounds)

    def __call__(self, X, Y=None, eval_gradient=False):
        ls = np.asarray(self.length_scale, dtype=np.float64)
        ls = ls if self.anisotropic else float(ls.reshape(-1)[0])
        X = np.atleast_2d(X)
        if Y is None:
            Y = X
        elif eval_gradient:
            raise ValueError("gradient only when Y is None")
        ind = np.expand_dims(X, axis=1) != Y
        K = np.exp(-np.sum(ls * ind, axis=2))
        if not eval_gradient:
            return K
        if self.anisotropic:
            grad = -np.expand_dims(K, -1) * ind * ls
        else:
            grad = -np.expand_dims(K * np.sum(ind, axis=2), -1) * ls
        return K, grad


class RecordingGPR(GaussianProcessRegressor):
    def _constrained_optimization(self, obj_func, initial_theta, bounds):
        theta, fmin = super()._constrained_optimization(obj_func, initial_theta, bounds)
        self.record_.append((np.array(initial_theta, dtype=np.float64), np.array(theta, dtype=np.float64), float(fmin)))
        return theta, fmin


def _codes(r, N, cats):
    return np.stack([r.integers(0, c, N) for c in cats], axis=1).astype(np.float64)


def cases():
    """(name, categories per dimension, codes, y, random_state)."""
    r = np.random.default_rng(77)
    out = []

    def effect(c):
        return r.standard_normal(c)

    for name, cats, N, w, noise, rs in (
            ("c3_d1_n20", [3], 20, [1.0], 0.1, 3),
            ("c7_d1_n60", [7], 60, [1.0], 0.2, 5),
            ("c2_d1_n16", [2], 16, [1.0], 0.3, 9),
            ("mixed_d3_n100", [2, 3, 7], 100, [1.0, 0.5, 2.0], 0.1, 11),
            ("one_d3_n80", [1, 3, 7], 80, [0.0, 1.0, 1.0], 0.1, 13),
            ("flat_d3_n40", [3, 7, 2], 40, [1.0, 0.7, 0.0], 0.05, 17),
            ("mixed_d8_n512", [1, 2, 3, 7, 2, 3, 7, 3], 512, [0, 1.0, 0.5, 1.5, 0, 0, 0.8, 0], 0.1, 19),
            ("noisy_d8_n200", [2, 3, 7, 7, 3, 2, 3, 7], 200, [1.0, 1.0, 0.5, 0.3, 0.2, 0.4, 1.0, 0.6], 0.8, 23)):
        X = _codes(r, N, cats)
        eff = [effect(c) for c in cats]
        y = sum(wj * e[X[:, j].astype(int)] for j, (wj, e) in enumerate(zip(w, eff)))
        y = y + 0.3 * (eff[-1][X[:, -1].astype(int)] * eff[0][X[:, 0].astype(int)]) * (len(cats) > 1)
        y = np.asarray(y, dtype=np.float64) + noise * r.standard_normal(N)
        Xc = np.concatenate([X[:20], _codes(r, 280, cats)])        # candidates: 20 training points and 280 draws
        out.append((name, np.array(cats), X, y, Xc, rs))
    return out


def main():
    out = {}
    for name, cats, X, y, Xc, random_state in cases():
        D = X.shape[1]
        seed = estimator_seed(random_state)
        kernel = ConstantKernel(1.0, (0.01, 1000.0)) * Hamming(length_scale=np.ones(D)) + WhiteKernel()
        gpr = RecordingGPR(kernel=kernel, alpha=1e-10, normalize_y=True, n_restarts_optimizer=2, random_state=seed)
        gpr.record_ = []
        gpr.fit(X, y)
        rec = gpr.record_
        probes = np.stack([a for a, _, _ in rec] + [gpr.kernel_.theta])
        lg = [gpr.log_marginal_likelihood(t, eval_gradient=True, clone_kernel=True) for t in probes]
        kernel_theta = gpr.kernel_.theta.copy()
        gpr.kernel_.set_params(k2__noise_level=0.0)                 # skopt's predict-time hack [RECALL]
        mu, sd = gpr.predict(Xc, return_std=True)
        out[name] = dict(categories=cats, X=X, y=y, Xc=Xc, random_state=random_state, seed=seed,
                         theta0=np.stack([a for a, _, _ in rec]), theta=np.stack([b for _, b, _ in rec]),
                         neg_lml=np.array([c for _, _, c in rec]), kernel_theta=kernel_theta, lml=gpr.log_marginal_likelihood_value_,
                         probe_theta=probes, probe_lml=np.array([v for v, _ in lg]), probe_grad=np.stack([g for _, g in lg]),
                         mu=mu, std=sd)
        print(f"{name}: winner {int(np.argmin(out[name]['neg_lml']))} lml {gpr.log_marginal_likelihood_value_:.6f} "
              f"θ {np.round(kernel_theta, 4)}")
    path = os.path.join(ROOT, "tests", "golden", "hamming_cases.npz")
    np.savez_compressed(path, sklearn_version=sklearn.__version__, names=np.array(sorted(out)),
                        **{f"{k}__{f}": v[f] for k, v in out.items() for f in v})
    print(path)


if __name__ == "__main__":
    main()
