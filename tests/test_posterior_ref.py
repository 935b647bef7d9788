"""CPU: pin tests/_posterior_ref.py — the torch FP64 posterior test_gpu_grid_scale.py measures the engine against — to the real
scikit-learn golden vectors (the tolerances of test_oracle.py) and to oracle.suggest to 1e-12, on candidates that are exact
copies of trials or within 1e-7 of one, where a distance formed as ‖a‖² + ‖b‖² − 2a·b would cancel."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O
from tests import _posterior_ref as R

RTOL = 1e-12


def _golden_posterior(g, **kw):
    return R.posterior(g["X"], g["y"], g["Xc"], kind=g["kind"], length_scale=g["length_scale"], amplitude=g["amplitude"],
                       noise=g["noise"], xi=g["xi"], kappa=g["kappa"], device="cpu", **kw)


def test_reference_matches_sklearn_golden(golden):
    r = _golden_posterior(golden)
    f = r["fit"]
    np.testing.assert_allclose(f["L"].numpy(), golden["L"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(f["alpha"].numpy(), golden["alpha"], rtol=1e-7, atol=1e-9)
    assert abs(f["y_mean"] - golden["y_mean"]) < 1e-12 and abs(f["y_std"] - golden["y_std"]) < 1e-12
    np.testing.assert_allclose(r["mu"], golden["mu"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(r["std"], golden["std"], rtol=0, atol=1e-8)
    a = golden["acq_kind"]
    np.testing.assert_allclose(r["acq"][a], golden["acq"], rtol=0, atol=1e-9)
    assert r["top"][a][0] == golden["index"]
    assert abs(f["lml"] - golden["lml"]) < 1e-7 * max(1.0, abs(golden["lml"]))


def _near_trials(X, Xc, n, seed):
    """Xc with n rows replaced by exact copies of trials and n by trials moved by 1e-7·u, u uniform in [−1, 1)^D."""
    r = np.random.default_rng(seed)
    G = Xc.copy()
    rows = r.choice(len(Xc), 2 * n, replace=False)
    G[rows[:n]] = X[r.choice(len(X), n, replace=False)]
    G[rows[n:]] = X[r.choice(len(X), n, replace=False)] + 1e-7 * (2 * r.random((n, X.shape[1])) - 1)
    return G, rows


def _pi_atol(mu, std, y_opt, xi, tol):
    """The bound `tol` on μ and σ carried through PI = Φ(z), z = (y_opt − ξ − μ)/σ: |dPI| ≤ φ(z)·(|dμ| + |z|·|dσ|)/σ.  PI is the
    one acquisition whose derivative is not bounded (1/σ), so two FP64 evaluations of it agree only to that."""
    z = np.where(std > 0, (y_opt - xi - mu) / np.where(std > 0, std, 1.0), 0.0)
    return np.where(std > 0, np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi) * tol * (1 + np.abs(z)) / np.where(std > 0, std, 1.0), 0.0) + tol


# (kind, ARD, normalize_y, y = c + s·y₀) at the noise of record.  Two LAPACK builds agree to a fraction of eps·cond(K): 1e-12 holds
# for the Matérn fits (cond(K) 2.5e4 … 3.2e4, worst |dμ| 1.2e-12·y_std); the RBF Gram matrix is 5× worse conditioned (1.2e5 … 1.3e5)
# and its worst |dμ| is 1.9e-12·y_std, so RBF is held to 4e-12.  At noise 1e-6 the difference
# reaches 1e-10 — test_gpu_grid_scale.py measures that regime against its own bound.
TOL = {"matern52": RTOL, "rbf": 4e-12}
CASES = [("matern52", False, True, 0.0, 1.0), ("matern52", True, True, 2e4, 5.0), ("rbf", False, True, 0.0, 1.0), ("rbf", True, False, 0.0, 1.0)]


@pytest.mark.parametrize("kind,ard,normalize_y,c,s", CASES,
                         ids=[f"{k}-{'ard' if a else 'iso'}-{'norm' if ny else 'raw'}-y{c:g}" for k, a, ny, c, s in CASES])
def test_reference_matches_the_oracle_next_to_trials(kind, ard, normalize_y, c, s):
    """μ, σ, EI and LCB to 1e-12 of each quantity's scale (y_std) and relative, PI to that bound carried through Φ, and the same
    first-index argmax, at N = 300 with exact and 1e-7-near copies of trials in the grid."""
    noise = 1e-3
    N, M, D = 300, 2000, 6
    X, y0, Xc = O.synthetic(N, M, D)
    y = c + s * y0
    Xc, rows = _near_trials(X, Xc, 40, seed=N + D)
    th = O.theta_of_record(D)
    ls = th["length_scale"] * (np.linspace(0.5, 2.0, D) if ard else 1.0)
    kw = dict(kind=kind, length_scale=ls, amplitude=th["amplitude"], noise=noise, xi=th["xi"], kappa=th["kappa"])
    r = R.posterior(X, y, Xc, normalize_y=normalize_y, device="cpu", **kw)
    f = r["fit"]
    scale, tol = f["y_std"], TOL[kind]
    for acq in R.ACQS:
        o = O.suggest(X, y, Xc, acq=acq, normalize_y=normalize_y, **kw)
        if acq == "ei":
            for what in ("mu", "std"):
                d = np.abs(r[what] - o[what])
                print(f"\n{kind} ard={ard}: max|d {what}| / y_std {d.max() / scale:.2e} (near trials {d[rows].max() / scale:.2e})")
                np.testing.assert_allclose(r[what], o[what], rtol=tol, atol=tol * scale, err_msg=what)
            assert np.all(r["std"][rows[:40]] ** 2 <= noise * scale ** 2 * 1.0001)    # the trial copies: σ² below the noise level
        atol = _pi_atol(o["mu"], o["std"], f["y_opt"], kw["xi"], tol * scale) if acq == "pi" else tol * scale
        d = np.abs(r["acq"][acq] - o["acq"])
        assert np.all(d <= tol * np.abs(o["acq"]) + atol), (acq, int(np.argmax(d - atol)), float(d.max()))
        i, v, _ = r["top"][acq]
        assert i == o["index"] and abs(v - o["value"]) <= tol * max(scale, abs(o["value"])), (acq, i, v, o["index"], o["value"])
    assert abs(f["lml"] - o["fit"]["lml"]) <= tol * abs(o["fit"]["lml"])


def test_chunks_and_distance_slabs_do_not_change_the_result():
    """A budget small enough for one-row distance slabs and a few rows per chunk (ragged last chunk) gives the one-shot values:
    each row's arithmetic does not depend on the chunk it lands in, up to the row sums of V², which BLAS may order by width."""
    X, y, Xc = O.synthetic(130, 1001, 5)
    th = O.theta_of_record(5)
    kw = dict(kind="matern52", length_scale=th["length_scale"], amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96, device="cpu")
    one = R.posterior(X, y, Xc, **kw)
    small = R.posterior(X, y, Xc, budget=8 * 130 * 5 * 33, **kw)       # 33 rows per chunk, 8 per distance slab
    for what in ("mu", "std"):
        np.testing.assert_allclose(small[what], one[what], rtol=1e-14, atol=1e-15)
    assert small["top"] == one["top"]


def test_float32_candidates_are_widened():
    X, y, Xc = O.synthetic(64, 500, 4)
    th = O.theta_of_record(4)
    kw = dict(kind="rbf", length_scale=th["length_scale"], amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96, device="cpu")
    Xc32 = Xc.astype(np.float32)
    a = R.posterior(X, y, Xc32, **kw)
    b = R.posterior(X, y, torch.tensor(Xc32), **kw)
    c = R.posterior(X, y, Xc32.astype(np.float64), **kw)
    for what in ("mu", "std"):
        assert np.array_equal(a[what], c[what]) and np.array_equal(b[what], c[what])


@pytest.mark.parametrize("N,P", [(300, 128), (300, 1024), (2048, 1024)])
def test_prefix_variance_against_the_oracle_inverse(N, P):
    """predict_normalised: μ_n and σ²_n are the oracle's posterior in normalised units, σ²_P at P ≥ N is σ²_n, σ²_P never
    increases with P, and σ²_P is amplitude − ‖(L⁻¹)[:P, :P] k*[:P]‖² with L the oracle's factor — the first P rows of L⁻¹ are
    those of the inverse of L[:P, :P], so the prefix variance is the posterior given the first P trials."""
    X, y, Xc = O.synthetic(N, 400, 6)
    th = O.theta_of_record(6)
    kw = dict(length_scale=th["length_scale"], amplitude=1.7, noise=1e-3)
    f = R.fit(X, y, kind="matern52", device="cpu", **kw)
    Ps = sorted({1, 64, P, N // 2, N})
    r = R.predict_normalised(f, Xc, prefixes=Ps)
    o = O.gp_fit(X, y, kind="matern52", **kw)
    mu, sd = O.gp_predict(o, Xc)
    np.testing.assert_allclose(r["mu_n"], (mu - o["y_mean"]) / o["y_std"], rtol=0, atol=1e-11)   # 2.4e-12 at N = 2048
    np.testing.assert_allclose(np.maximum(r["var_n"], 0.0), (sd / o["y_std"]) ** 2, rtol=0, atol=1e-12)
    assert np.array_equal(r["var_p"][N], r["var_n"])
    for a, b in zip(Ps[:-1], Ps[1:]):
        assert np.all(r["var_p"][b] <= r["var_p"][a] + 1e-14), (a, b)
    p = min(P, N)
    Ks = O.kernel_matrix(Xc, X[:p], kw["length_scale"], "matern52", kw["amplitude"])
    Winv = np.linalg.inv(np.tril(o["L"][:p, :p]))
    ref = kw["amplitude"] - ((Ks @ Winv.T) ** 2).sum(1)
    np.testing.assert_allclose(r["var_p"][P], ref, rtol=0, atol=1e-11)
    assert np.all(r["var_p"][P] >= r["var_n"] - 1e-14)
