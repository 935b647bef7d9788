"""CPU: pin oracle/gp_oracle.py against the golden vectors produced by the real scikit-learn GPR
(oracle/make_golden.py) and against self-authored known-answer checks (SURVEY.md §8(c) item 3)."""
import os

import numpy as np
import pytest

from oracle import gp_oracle as O


def _suggest(g, **over):
    kw = dict(kind=g["kind"], length_scale=g["length_scale"], amplitude=g["amplitude"], noise=g["noise"],
              acq=g["acq_kind"], xi=g["xi"], kappa=g["kappa"])
    kw.update(over)
    return O.suggest(g["X"], g["y"], g["Xc"], **kw)


def test_oracle_matches_sklearn_golden(golden):
    r = _suggest(golden)
    np.testing.assert_allclose(r["fit"]["L"], golden["L"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(r["fit"]["alpha"], golden["alpha"], rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(r["mu"], golden["mu"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(r["std"], golden["std"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(r["acq"], golden["acq"], rtol=0, atol=1e-9)
    assert r["index"] == golden["index"]
    assert abs(r["fit"]["lml"] - golden["lml"]) < 1e-7 * max(1.0, abs(golden["lml"]))


def test_n1_closed_form():
    # one trial: mu_n(x) = k(x,x1)·y1/(1+s²) with y normalised to 0 => mean is y1; var = 1 − k²/(1+s²)
    x1 = np.array([[0.3, 0.6]]); y1 = np.array([1.7]); Xc = np.random.default_rng(0).random((50, 2))
    fit = O.gp_fit(x1, y1, kind="rbf", length_scale=0.5, noise=1e-3)
    mu, std = O.gp_predict(fit, Xc)
    k = O.kernel_matrix(Xc, x1, 0.5, "rbf")[:, 0]
    np.testing.assert_allclose(mu, 1.7, atol=1e-12)
    np.testing.assert_allclose(std ** 2, 1 - k * k / (1 + 1e-3), atol=1e-12)


def test_candidate_equals_training_point_variance():
    X, y, Xc = O.synthetic(40, 10, 3)
    th = O.theta_of_record(3)
    fit = O.gp_fit(X, y, kind="matern52", length_scale=th["length_scale"], noise=th["noise"])
    mu, std = O.gp_predict(fit, X[:5])
    # posterior variance at a training point is below the noise level, and tiny vs. the prior (1)
    assert np.all(std ** 2 <= th["noise"] * fit["y_std"] ** 2 * 1.0001)


def test_permutation_and_shard_invariance():
    X, y, Xc = O.synthetic(64, 300, 4)
    th = O.theta_of_record(4)
    kw = dict(kind="matern52", length_scale=th["length_scale"], noise=th["noise"])
    a = O.suggest(X, y, Xc, **kw)
    p = np.random.default_rng(5).permutation(64)
    b = O.suggest(X[p], y[p], Xc, **kw)
    np.testing.assert_allclose(a["acq"], b["acq"], atol=1e-10)
    # sharding the grid: max over shards with lowest-global-index tie-break == global first argmax
    best = None
    for r in range(4):
        s = O.suggest(X, y, Xc[r * 75:(r + 1) * 75], **kw)
        cand = (s["value"], -(r * 75 + s["index"]))
        best = cand if best is None or cand > best else best
    assert -best[1] == a["index"]


def test_duplicate_candidate_lowest_index_wins():
    X, y, Xc = O.synthetic(32, 128, 3)
    th = O.theta_of_record(3)
    kw = dict(kind="rbf", length_scale=th["length_scale"], noise=th["noise"])
    i = O.suggest(X, y, Xc, **kw)["index"]
    Xd = np.concatenate([Xc, Xc[i:i + 1], Xc[i:i + 1]])
    assert O.suggest(X, y, Xd, **kw)["index"] == i
    j = 0 if i != 0 else 1
    Xe = Xc.copy(); Xe[j] = Xc[i]
    assert O.suggest(X, y, Xe, **kw)["index"] == min(i, j)


def test_properties():
    X, y, Xc = O.synthetic(100, 500, 5)
    th = O.theta_of_record(5)
    r = O.suggest(X, y, Xc, kind="matern52", length_scale=th["length_scale"], noise=th["noise"])
    K = O.kernel_matrix(X, X, th["length_scale"], "matern52")
    assert np.allclose(K, K.T) and np.linalg.eigvalsh(K).min() > -1e-10
    L = r["fit"]["L"]
    np.testing.assert_allclose(L @ L.T, K + th["noise"] * np.eye(100), atol=1e-12)
    assert (r["std"] >= 0).all() and (r["acq"] >= 0).all()
    # EI -> 0 when sigma -> 0 and mu > y_opt
    assert O.acquisition(np.array([2.0]), np.array([1e-12]), 1.0)[0] < 1e-300 + 1e-12
    assert O.acquisition(np.array([2.0]), np.array([0.0]), 1.0)[0] == 0.0


def test_lml_gradient_matches_sklearn_golden():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "lmlgrad_cases.npz"), allow_pickle=False)
    names = sorted({k.split("__")[0] for k in z.files})
    assert len(names) == 4
    for n in names:
        ls = z[f"{n}__ls"]
        for chunk in (1, 7, 64):
            lml, g = O.lml_and_grad(z[f"{n}__X"], z[f"{n}__y"], kind=str(z[f"{n}__kind"]), length_scale=ls if len(ls) > 1 else float(ls[0]),
                                    amplitude=float(z[f"{n}__amp"]), noise=float(z[f"{n}__noise"]), chunk=chunk)
            assert abs(lml - float(z[f"{n}__lml"])) < 1e-9
            np.testing.assert_allclose(g, z[f"{n}__grad"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("n,D,kind,ard", [(150, 3, "matern52", False), (97, 17, "rbf", True), (130, 33, "matern52", True), (1, 2, "rbf", False)])
def test_lml_gradient_row_chunks_sum_to_the_one_shot_gradient(n, D, kind, ard):
    """The row-chunked gradient (what makes N = 8192, D = 32 fit in memory) is the one-shot (n, n, D) computation up to the
    summation order, whatever the chunk and however the last chunk is cut."""
    r = np.random.default_rng(n * D)
    X, y = r.random((n, D)), r.standard_normal(n)
    ls = 0.3 * np.sqrt(D) * (np.linspace(0.7, 1.4, D) if ard else 1.0)
    kw = dict(kind=kind, length_scale=ls, amplitude=1.3, noise=1e-3)
    lml0, g0 = O.lml_and_grad(X, y, chunk=n, **kw)
    for chunk in (1, 7, 64):
        lml, g = O.lml_and_grad(X, y, chunk=chunk, **kw)
        assert lml == lml0
        np.testing.assert_allclose(g, g0, rtol=1e-12, atol=1e-12 * np.abs(g0).max())


@pytest.mark.parametrize("N", [4096, 5800])
def test_not_pd_constructions_fail_exactly_at_the_chosen_pivot_in_lapack(N):
    """oracle.not_pd_at(N, p): LAPACK's dpotrf on the RBF Gram matrix (amplitude 1, ℓ = 1, noise 0) reports the first
    non-positive pivot at exactly p — the histories the GPU tests use to pin the engine's `info`."""
    from scipy.linalg import lapack
    for p in (2, 64, 65, 256, 257, 2985, N):
        X, _ = O.not_pd_at(N, p)
        assert np.all(X == np.round(X))
        K = O.kernel_matrix(X, X, 1.0, "rbf", 1.0)
        _, info = lapack.dpotrf(K, lower=1, clean=0, overwrite_a=1)
        assert info == p, (N, p, info)
    X, _ = O.not_pd_at(N, 2985)
    K = O.kernel_matrix(X[:2984], X[:2984], 1.0, "rbf", 1.0)
    _, info = lapack.dpotrf(K, lower=1, clean=0, overwrite_a=1)
    assert info == 0
