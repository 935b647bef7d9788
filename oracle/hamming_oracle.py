"""FP64 NumPy restatement of skopt's GP on an all-categorical space (test infrastructure only).

It works on category codes, straight from the Hamming formula, and never through the one-hot columns the engine uses, so it
checks ``kubeflow_b200.hamming``'s mapping rather than repeating it.  Items marked [RECALL] restate skopt from memory (skopt
is not a dependency of this project); where they and tests/golden/hamming_cases.npz (made by the real scikit-learn
GaussianProcessRegressor) disagree, the data wins.

* [RECALL] ``skopt.utils.cook_estimator("GP", space)`` with ``space.is_categorical``: ``ConstantKernel(1.0, (0.01, 1000.0)) *
  HammingKernel(length_scale=np.ones(n_dims))``, ``normalize_y=True``, ``noise="gaussian"`` (a ``WhiteKernel()`` is added:
  noise 1.0, bounds (1e-5, 1e5)), ``n_restarts_optimizer=2``; sklearn's ``alpha`` = 1e-10 sits on the diagonal with the noise.
* [RECALL] ``HammingKernel``: ``k(x, y) = exp(−Σ_j l_j·[x_j ≠ y_j])``; ``l_j`` multiplies the mismatch.  Bounds (1e-5, 1e5);
  the fit works on log l_j.
* [RECALL] ``normalize_dimensions`` gives an all-categorical space the identity transform: the kernel compares the raw
  category values (codes here).
* [RECALL] skopt's GaussianProcessRegressor zeroes the WhiteKernel after the fit, so the predictive variance is
  amp − k*ᵀK⁻¹k* without the noise.

θ is in sklearn's order: (log amp, log l_1..D, log noise).  The acquisitions are ``oracle.gp_oracle``'s (they depend on μ and
σ only).
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_solve, cholesky, solve_triangular
from scipy.optimize import minimize

from oracle.gp_oracle import acquisition, first_argmax  # noqa: F401  (re-exported for the tests)

ALPHA = 1e-10
AMP_BOUNDS = (0.01, 1000.0)
L_BOUNDS = (1e-5, 1e5)
NOISE_BOUNDS = (1e-5, 1e5)


def log_bounds(D: int) -> np.ndarray:
    return np.log(np.array([AMP_BOUNDS] + [L_BOUNDS] * D + [NOISE_BOUNDS], dtype=np.float64))


def mismatch_sum(A, B, l) -> np.ndarray:
    """Σ_j l_j·[A_ij ≠ B_kj] for every row pair (i, k), dimension by dimension."""
    A, B = np.atleast_2d(A), np.atleast_2d(B)
    l = np.broadcast_to(np.asarray(l, dtype=np.float64), (A.shape[1],))
    S = np.zeros((A.shape[0], B.shape[0]))
    for j in range(A.shape[1]):
        S += l[j] * (A[:, j, None] != B[None, :, j])
    return S


def kernel(A, B, l, amp=1.0) -> np.ndarray:
    """amp · exp(−Σ_j l_j·[a_j ≠ b_j])."""
    return amp * np.exp(-mismatch_sum(A, B, l))


def _normalise(y):
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    m = float(np.mean(y))
    s = float(np.std(y))
    return (y - m) / (s if s != 0.0 else 1.0), m, (s if s != 0.0 else 1.0)


def fit(X, y, theta):
    """Cholesky factor, α and normalisation of the GP at θ (sklearn order).  Raises LinAlgError if K is not positive definite."""
    t = np.asarray(theta, dtype=np.float64)
    amp, l, noise = np.exp(t[0]), np.exp(t[1:-1]), np.exp(t[-1])
    yn, ym, ys = _normalise(y)
    Kh = kernel(X, X, l)
    K = amp * Kh
    K[np.diag_indices_from(K)] += noise + ALPHA
    Lc = cholesky(K, lower=True)
    alpha = cho_solve((Lc, True), yn)
    return dict(X=np.asarray(X), y=np.asarray(y, dtype=np.float64), amp=amp, l=l, noise=noise, Kh=Kh, L=Lc, alpha=alpha, yn=yn,
                y_mean=ym, y_std=ys)


def lml_and_grad(X, y, theta):
    """sklearn's log_marginal_likelihood(θ, eval_gradient=True): LML and ∂LML/∂θ in sklearn's order.
    ∂K/∂log amp = amp·Kh; ∂K/∂log l_j = −amp·Kh·l_j·[x_j ≠ y_j]; ∂K/∂log noise = noise·I (alpha is not a parameter)."""
    f = fit(X, y, theta)
    n = len(f["yn"])
    lml = -0.5 * f["yn"] @ f["alpha"] - np.log(np.diag(f["L"])).sum() - 0.5 * n * np.log(2 * np.pi)
    Kinv = cho_solve((f["L"], True), np.eye(n))
    T = np.outer(f["alpha"], f["alpha"]) - Kinv
    G = T * (f["amp"] * f["Kh"])
    Xa = np.atleast_2d(X)
    g = [0.5 * G.sum()]
    for j in range(Xa.shape[1]):
        g.append(-0.5 * f["l"][j] * G[Xa[:, j, None] != Xa[None, :, j]].sum())
    g.append(0.5 * f["noise"] * np.trace(T))
    return float(lml), np.array(g)


def objective(X, y, theta):
    """(−LML, −gradient); a θ whose Gram matrix is not positive definite is (+inf, 0), as in sklearn."""
    try:
        lml, g = lml_and_grad(X, y, theta)
    except np.linalg.LinAlgError:
        return np.inf, np.zeros(len(theta))
    return -lml, -g


def starts(D: int, seed: int, n_restarts: int = 2) -> np.ndarray:
    """log(1, …, 1), then n_restarts draws of RandomState(seed).uniform over the log bounds (sklearn's restarts)."""
    b = log_bounds(D)
    rng = np.random.RandomState(seed)
    return np.stack([np.zeros(D + 2)] + [rng.uniform(b[:, 0], b[:, 1]) for _ in range(n_restarts)])


def skopt_fit(X, y, *, seed, n_restarts=2, maxiter=None):
    """sklearn's restart search: SciPy's L-BFGS-B from each start in turn; the winner is np.argmin of the final −LML."""
    D = np.atleast_2d(X).shape[1]
    b = log_bounds(D)
    runs = []
    for x0 in starts(D, seed, n_restarts):
        r = minimize(lambda t: objective(X, y, t), x0, method="L-BFGS-B", jac=True, bounds=b,
                     options={} if maxiter is None else dict(maxiter=maxiter))
        runs.append(dict(theta0=x0, theta=np.asarray(r.x), neg_lml=float(r.fun), nit=int(r.nit), nfev=int(r.nfev)))
    w = int(np.argmin([r["neg_lml"] for r in runs]))
    return dict(theta=runs[w]["theta"], lml=-runs[w]["neg_lml"], winner=w, starts=runs)


def predict(f, Xc, batch=4096):
    """Posterior mean and std on the raw y scale at the rows of Xc (codes)."""
    Xc = np.atleast_2d(Xc)
    mu, sd = np.empty(len(Xc)), np.empty(len(Xc))
    for s in range(0, len(Xc), batch):
        Ks = kernel(Xc[s:s + batch], f["X"], f["l"], f["amp"])
        mu[s:s + batch] = f["y_mean"] + f["y_std"] * (Ks @ f["alpha"])
        V = solve_triangular(f["L"], Ks.T, lower=True)
        var = np.maximum(f["amp"] - np.einsum("ij,ij->j", V, V), 0.0)
        sd[s:s + batch] = f["y_std"] * np.sqrt(var)
    return mu, sd


def suggest(X, y, Xc, theta, acq="ei", xi=0.01, kappa=1.96):
    """One fit at θ and the first-index argmax of the acquisition over the candidate codes Xc."""
    f = fit(X, y, theta)
    mu, sd = predict(f, Xc)
    a = acquisition(mu, sd, float(np.min(f["y"])), acq, xi, kappa)
    i = first_argmax(a)
    return dict(index=i, value=float(a[i]), acq=a, mu=mu, std=sd, fit=f)
