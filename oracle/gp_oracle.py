"""CPU oracle for the Katib `bayesianoptimization` (scikit-optimize GP) suggestion hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``kubeflow_b200/`` may import this module; only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py`` do.  The product path is the CUDA library behind ``include/kbo.h`` and it fails
loudly when that library is missing.

PARITY UNPINNED BY THE REFERENCE.  ``/root/reference`` (kubeflow/kubeflow @ 6d6b78bc) holds no
Katib source, no proto and no test that reads a suggested value (SURVEY.md §0: the only
caller-side test, ``testing/katib_studyjob_test.py:196-206``, polls a StudyJob for "Running").
The arithmetic of the path lives in third-party code that the reference does not vendor or pin:
kubeflow/katib ``pkg/suggestion/v1beta1/skopt`` -> scikit-optimize (``Optimizer.tell/ask``,
``skopt.acquisition.gaussian_{ei,lcb,pi}``) -> scikit-learn ``GaussianProcessRegressor``.
scikit-optimize is not installable here; scikit-learn 1.9.0 *is* importable, so this file is a
plain NumPy/SciPy fp64 restatement of the published algorithm (Rasmussen & Williams Alg. 2.1 as
coded in scikit-learn); it is pinned against the real ``sklearn.gaussian_process.GaussianProcessRegressor``
run in this container: the golden vectors are committed under ``tests/golden/`` (generators:
``oracle/make_golden.py``, ``oracle/make_golden_lmlgrad.py``) and checked by ``tests/test_oracle.py``.

Line references: ``$SK`` = site-packages/sklearn/gaussian_process (scikit-learn 1.9.0).
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import cholesky, cho_solve, solve_triangular
from scipy.spatial.distance import cdist
from scipy.special import ndtr

KERNEL_RBF = "rbf"
KERNEL_MATERN52 = "matern52"
ACQ_EI = "ei"
ACQ_LCB = "lcb"
ACQ_PI = "pi"


def kernel_matrix(A, B, length_scale, kind=KERNEL_MATERN52, amplitude=1.0):
    """amplitude * k(A, B) for the two kernels on the path.

    RBF:        $SK/kernels.py:1559-1570  (X/ℓ, sqeuclidean cdist, exp(-d²/2))
    Matern-5/2: $SK/kernels.py:1713-1729  (X/ℓ, euclidean cdist, K=√5·d, (1+K+K²/3)·exp(-K))
    Product with ConstantKernel: $SK/kernels.py:971, :1278 (skopt: ``cov_amplitude * Matern``).
    ``length_scale`` is a scalar or a length-D vector (anisotropic / ARD).
    """
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    ls = np.asarray(length_scale, dtype=np.float64)
    if kind == KERNEL_RBF:
        d2 = cdist(A / ls, B / ls, metric="sqeuclidean")
        K = np.exp(-0.5 * d2)
    elif kind == KERNEL_MATERN52:
        d = cdist(A / ls, B / ls, metric="euclidean")
        s = d * np.sqrt(5.0)
        K = (1.0 + s + s * s / 3.0) * np.exp(-s)
    else:
        raise ValueError(f"unknown kernel {kind!r}")
    return amplitude * K


def gp_fit(X, y, *, kind=KERNEL_MATERN52, length_scale=1.0, amplitude=1.0, noise=1e-10,
           normalize_y=True):
    """Fixed-θ GaussianProcessRegressor.fit ($SK/_gpr.py:233-368 with optimizer=None).

    normalize_y: :275-280 (mean / std with the zero-std guard of _handle_zeros_in_scale).
    K = k(X,X); K[diag] += alpha: :349-350.   L = cholesky(K, lower): :352.
    alpha_ = cho_solve(L, y): :363.
    """
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    if normalize_y:
        y_mean = float(np.mean(y))
        y_std = float(np.std(y))
        if y_std < 10 * np.finfo(np.float64).eps:  # sklearn.preprocessing._data._handle_zeros_in_scale
            y_std = 1.0
    else:
        y_mean, y_std = 0.0, 1.0
    yn = (y - y_mean) / y_std
    K = kernel_matrix(X, X, length_scale, kind, amplitude)
    K[np.diag_indices_from(K)] += noise
    L = cholesky(K, lower=True, check_finite=False)
    alpha = cho_solve((L, True), yn, check_finite=False)
    # log marginal likelihood at fixed θ ($SK/_gpr.py:604-618) — reported, not on the argmax path
    lml = float(-0.5 * yn @ alpha - np.log(np.diag(L)).sum() - 0.5 * len(yn) * np.log(2 * np.pi))
    return dict(X=X, y=y, yn=yn, y_mean=y_mean, y_std=y_std, L=L, alpha=alpha, kind=kind,
                length_scale=np.asarray(length_scale, dtype=np.float64), amplitude=float(amplitude),
                noise=float(noise), lml=lml)


def gp_predict(fit, Xc, batch=8192):
    """GaussianProcessRegressor.predict(return_std=True) ($SK/_gpr.py:445-500), row-batched.

    K* = k(Xc, X): :446.  mean = K*·alpha_: :447, un-normalise :450.
    V = solve_triangular(L, K*ᵀ): :460.  var = diag − Σ V²: :480-481, clamp <0 → 0: :485-491,
    × y_std²: :494, sqrt: :500.   kernel_.diag(X) of C*Matern / C*RBF is ``amplitude``
    ($SK/kernels.py:490 for the stationary part).
    """
    Xc = np.asarray(Xc, dtype=np.float64)
    M = Xc.shape[0]
    mu = np.empty(M)
    std = np.empty(M)
    for s in range(0, M, batch):
        Ks = kernel_matrix(Xc[s:s + batch], fit["X"], fit["length_scale"], fit["kind"], fit["amplitude"])
        m = Ks @ fit["alpha"]
        V = solve_triangular(fit["L"], Ks.T, lower=True, check_finite=False)
        var = fit["amplitude"] - np.einsum("ij,ij->j", V, V)
        var[var < 0] = 0.0
        mu[s:s + batch] = fit["y_std"] * m + fit["y_mean"]
        std[s:s + batch] = np.sqrt(var * fit["y_std"] ** 2)
    return mu, std


def acquisition(mu, std, y_opt, acq=ACQ_EI, xi=0.01, kappa=1.96):
    """Acquisition value TO MAXIMISE (skopt returns the negation and argmins; same argument).

    EI  (skopt.acquisition.gaussian_ei):  imp = y_opt − ξ − μ; z = imp/σ; EI = imp·Φ(z) + σ·φ(z)
         where σ > 0, else 0.
    PI  (gaussian_pi): Φ(z) where σ > 0, else 0.
    LCB (gaussian_lcb): μ − κσ is minimised, so the value returned here is −(μ − κσ).
    """
    mu = np.asarray(mu, dtype=np.float64)
    std = np.asarray(std, dtype=np.float64)
    if acq == ACQ_LCB:
        return -(mu - kappa * std)
    out = np.zeros_like(mu)
    mask = std > 0
    imp = y_opt - xi - mu[mask]
    z = imp / std[mask]
    if acq == ACQ_EI:
        pdf = np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi)
        out[mask] = imp * ndtr(z) + std[mask] * pdf
    elif acq == ACQ_PI:
        out[mask] = ndtr(z)
    else:
        raise ValueError(f"unknown acquisition {acq!r}")
    return out


def first_argmax(values):
    """``np.argmin(-values)`` = first maximal index (skopt ``Optimizer._tell``: X_cand[argmin])."""
    return int(np.argmax(values))


def suggest(X, y, Xc, *, kind=KERNEL_MATERN52, length_scale=1.0, amplitude=1.0, noise=1e-10,
            acq=ACQ_EI, xi=0.01, kappa=1.96, normalize_y=True, batch=8192):
    """One ``tell`` + ``ask`` at fixed θ with acq_optimizer="sampling" over the candidate set Xc.

    y_opt = min(y) on the raw scale (skopt ``Optimizer._tell``: ``y_opt=np.min(self.yi)``).
    Returns dict(index, value, acq, mu, std, fit).
    """
    fit = gp_fit(X, y, kind=kind, length_scale=length_scale, amplitude=amplitude, noise=noise,
                 normalize_y=normalize_y)
    mu, std = gp_predict(fit, Xc, batch=batch)
    a = acquisition(mu, std, float(np.min(fit["y"])), acq, xi, kappa)
    i = first_argmax(a)
    return dict(index=i, value=float(a[i]), acq=a, mu=mu, std=std, fit=fit)


# ---------------------------------------------------------------------------------------------
# synthetic workload of record (SURVEY.md §8(d), BASELINE.md §3) — shared by tests and bench.py
# ---------------------------------------------------------------------------------------------
def synthetic(N, M, D, *, m_offset=0, m_total=None):
    """X = rng(1234).random((N,D)); y = sin(3·Σx/√D) + 0.1·rng(1235).normal; Xc = rng(4321).random((M,D)).

    ``m_offset``/``m_total`` give the row block a rank owns when the grid is sharded (§8(e)).
    """
    X = np.random.default_rng(1234).random((N, D))
    y = np.sin(3.0 * X.sum(axis=1) / np.sqrt(D)) + 0.1 * np.random.default_rng(1235).standard_normal(N)
    total = M if m_total is None else m_total
    Xc = np.random.default_rng(4321).random((total, D))[m_offset:m_offset + M]
    return X, y, Xc


def theta_of_record(D):
    """amplitude 1, ℓ_d = 0.3·√D, noise 1e-3, ξ = 0.01, κ = 1.96 (SURVEY.md §8(d))."""
    return dict(length_scale=0.3 * np.sqrt(D), amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96)


def lml_and_grad(X, y, *, kind=KERNEL_MATERN52, length_scale=1.0, amplitude=1.0, noise=1e-10, normalize_y=True, chunk=64):
    """Log-marginal likelihood and its gradient w.r.t. θ = (log amplitude, log noise, log ℓ_1..ℓ_P) at fixed data
    ($SK/_gpr.py:541-655: ``0.5·einsum((ααᵀ − K⁻¹), ∂K/∂θ)``; kernel gradients $SK/kernels.py:1571-1591 (RBF),
    :1731-1745 (Matérn ν=2.5), :1296 (Constant), :1421 (White)).  P = 1 (isotropic) or D.

    The (n, n, D) tensor of squared differences is formed ``chunk`` rows at a time (O(chunk·n·D) memory instead of 17 GB at
    n = 8192, D = 32); ``chunk >= n`` is the one-shot computation.  Only the summation order depends on ``chunk``."""
    fit = gp_fit(X, y, kind=kind, length_scale=length_scale, amplitude=amplitude, noise=noise, normalize_y=normalize_y)
    Xs = fit["X"] / fit["length_scale"]
    n, D = Xs.shape
    Kinv = cho_solve((fit["L"], True), np.eye(n), check_finite=False)
    g_amp, per_dim = 0.0, np.zeros(D)
    for s0 in range(0, n, chunk):
        G = np.outer(fit["alpha"][s0:s0 + chunk], fit["alpha"]) - Kinv[s0:s0 + chunk]
        diff2 = (Xs[s0:s0 + chunk, None, :] - Xs[None, :, :]) ** 2     # (chunk, n, D) scaled squared differences
        r2 = diff2.sum(-1)
        if kind == KERNEL_RBF:
            k = np.exp(-0.5 * r2)
            q = k                                              # ∂k/∂log ℓ_d = k · Δ_d²
        else:
            s = np.sqrt(5.0 * r2)
            k = (1 + s + s * s / 3) * np.exp(-s)
            q = (5.0 / 3.0) * (1 + s) * np.exp(-s)             # ∂k/∂log ℓ_d = (5/3)(1+s)e^{-s} · Δ_d²
        g_amp += 0.5 * np.sum(G * (amplitude * k))
        per_dim += 0.5 * amplitude * np.einsum("ij,ij,ijd->d", G, q, diff2)
    g_noise = 0.5 * noise * (np.sum(fit["alpha"] ** 2) - np.trace(Kinv))
    g_ls = per_dim if np.ndim(length_scale) and len(np.atleast_1d(length_scale)) > 1 else np.array([per_dim.sum()])
    return fit["lml"], np.concatenate([[g_amp, g_noise], g_ls])


def not_pd_at(N, p, *, isolated=None):
    """A history (X, y) in D = 4 whose RBF Gram matrix (amplitude 1, ℓ = 1, noise 0) has its first non-positive Cholesky pivot
    EXACTLY at the 1-based index p (2 <= p <= N), in any summation order:
      * the rows form part of the integer lattice {0, 2, …, 16}⁴ (spacing 2ℓ): a Kronecker product of 1-D factors whose smallest
        eigenvalue is ≈ 1 − 2e⁻² ≈ 0.73, so every principal submatrix has λ_min ≳ 0.28 even without noise;
      * row ``isolated`` (default (p − 1)//2) sits ≥ 64ℓ from every lattice point: exp(−d²/2) is exactly 0 in FP64 (and flushes to
        0 on the device), so its pivot is k(0) = 1 exactly, and its column of L is 1 on the diagonal, 0 elsewhere;
      * row p − 1 duplicates it: its pivot is 1 − 1·1 = 0 exactly.
    Integer coordinates make every squared distance exact."""
    assert 2 <= p <= N
    i = (p - 1) // 2 if isolated is None else isolated
    assert 0 <= i < p - 1
    g = np.arange(0, 18, 2, dtype=np.float64)
    lattice = np.stack(np.meshgrid(g, g, g, g, indexing="ij"), -1).reshape(-1, 4)
    lattice = lattice[np.random.default_rng(N * 7919 + p).permutation(len(lattice))]
    assert N - 2 <= len(lattice), f"N <= {len(lattice) + 2}"
    far = np.full(4, 1000.0)
    X = np.concatenate([lattice[:i], far[None], lattice[i:p - 2], far[None], lattice[p - 2:N - 2]])
    y = np.sin(X.sum(axis=1) / 8.0)
    return X, y
