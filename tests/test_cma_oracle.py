"""CPU: known-answer / property checks pinning oracle/cma_oracle.py (no upstream golden vectors exist offline)."""
import numpy as np

from oracle import cma_oracle as C


def test_parameters_match_tutorial_defaults():
    p = C.CmaParams(10, 4 + int(3 * np.log(10)))          # λ = 10 for n = 10 (tutorial eq. 48)
    assert p.popsize == 10 and p.mu == 5
    assert abs(p.weights[:p.mu].sum() - 1.0) < 1e-12 and (p.weights[:p.mu] > 0).all() and (p.weights[p.mu:] <= 0).all()
    assert np.all(np.diff(p.weights[:p.mu]) < 0)
    assert abs(p.mu_eff - 1.0 / (p.weights[:p.mu] ** 2).sum()) < 1e-12     # μ_eff = 1/Σw² for normalised positive weights
    assert 0 < p.c1 < p.cmu < 1 and p.c1 + p.cmu <= 1
    assert abs(p.chi_n - np.sqrt(10) * (1 - 1 / 40 + 1 / 2100)) < 1e-15
    # negative weights sum to -min(alpha_mu, alpha_mueff, alpha_posdef): keeps C positive definite (tutorial eq. 53)
    assert p.c1 + p.cmu * p.weights.sum() >= -1e-12


def test_update_is_rotation_equivariant():
    """CMA-ES is invariant under orthogonal transforms of the search space: rotating the steps rotates the state."""
    r = np.random.default_rng(0)
    n, lam = 6, 12
    Q, _ = np.linalg.qr(r.standard_normal((n, n)))
    z = r.standard_normal((lam, n))
    f = r.standard_normal(lam)
    a, b = C.CmaState(np.zeros(n), 0.7, lam), C.CmaState(np.zeros(n), 0.7, lam)
    _, Ya = C.ask(a, z)
    C.tell(a, Ya, f)
    C.tell(b, Ya @ Q.T, f)
    np.testing.assert_allclose(b.mean, Q @ a.mean, atol=1e-12)
    np.testing.assert_allclose(b.C, Q @ a.C @ Q.T, atol=1e-12)
    np.testing.assert_allclose(b.p_sigma, Q @ a.p_sigma, atol=1e-12)
    assert abs(a.sigma - b.sigma) < 1e-12


def test_converges_on_sphere_and_keeps_C_spd():
    r = np.random.default_rng(1)
    n, lam = 8, 16
    s = C.CmaState(np.full(n, 3.0), 2.0, lam)
    for g in range(150):
        X, Y = C.ask(s, r.standard_normal((lam, n)))
        C.tell(s, Y, C.sphere(X))
        assert np.linalg.eigvalsh((s.C + s.C.T) / 2).min() > 0
    assert C.sphere(s.mean[None])[0] < 1e-8 and s.sigma < 1e-3


def test_ties_broken_by_sample_index():
    s1, s2 = C.CmaState(np.zeros(3), 1.0, 6), C.CmaState(np.zeros(3), 1.0, 6)
    z = np.random.default_rng(2).standard_normal((6, 3))
    _, Y = C.ask(s1, z)
    C.tell(s1, Y, np.array([1.0, 0.0, 0.0, 2.0, 0.0, 3.0]))
    C.tell(s2, Y[[1, 2, 4, 0, 3, 5]], np.array([0.0, 0.0, 0.0, 1.0, 2.0, 3.0]))
    np.testing.assert_allclose(s1.mean, s2.mean, atol=1e-15)


def test_parameters_match_the_tutorial_formulas_evaluated_independently():
    """tests/golden/cma_known_answers.json: Hansen's parameter formulas evaluated with `decimal` (oracle/make_golden_cma.py) — for
    n = 10, λ = 10 these are the tutorial's default setting: w_1..5 = 0.4563, 0.2708, 0.1622, 0.0852, 0.0255, μ_eff = 3.167."""
    import json, os
    from tests.conftest import GOLDEN_DIR
    cases = json.load(open(os.path.join(GOLDEN_DIR, "cma_known_answers.json")))["cases"]
    assert abs(cases[0]["mu_eff"] - 3.1672992) < 1e-6 and abs(cases[0]["weights_first8"][0] - 0.45627265) < 1e-7   # the published 4-digit values
    for g in cases:
        p = C.CmaParams(g["n"], g["popsize"])
        for k in ("mu_eff", "c1", "cmu", "c_sigma", "d_sigma", "cc", "chi_n"):
            assert abs(getattr(p, k) - g[k]) <= 1e-13 * max(1.0, abs(g[k])), (g["n"], k, getattr(p, k), g[k])
        np.testing.assert_allclose(p.weights[:8], g["weights_first8"], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(p.weights[-2:], g["weights_last2"], rtol=1e-13, atol=1e-15)
        assert abs(p.weights.sum() - g["weights_sum"]) < 1e-12


def test_oracle_replays_its_committed_run_bit_for_bit():
    """tests/golden/cma_replay.npz: 12 seeded generations on the sphere and on Rastrigin.  Any change to the oracle's arithmetic
    (and hence to what the GPU sampler is compared with) shows up here first."""
    import os
    from tests.conftest import GOLDEN_DIR
    z = np.load(os.path.join(GOLDEN_DIR, "cma_replay.npz"))
    for name, f in (("sphere", C.sphere), ("rastrigin", C.rastrigin)):
        r = np.random.default_rng(20240917)
        st = C.CmaState(np.full(5, 1.5), 0.8, 8)
        for g in range(12):
            X, Y = C.ask(st, r.standard_normal((8, 5)))
            C.tell(st, Y, f(X))
            np.testing.assert_allclose(st.mean, z[f"{name}_mean"][g], rtol=0, atol=1e-13)
            np.testing.assert_allclose(st.C, z[f"{name}_C"][g], rtol=0, atol=1e-13)
            assert abs(st.sigma - z[f"{name}_sigma"][g]) <= 1e-13
            np.testing.assert_allclose(st.p_sigma, z[f"{name}_p_sigma"][g], rtol=0, atol=1e-13)
            np.testing.assert_allclose(st.pc, z[f"{name}_pc"][g], rtol=0, atol=1e-13)


def test_eigen_floors_only_non_positive_eigenvalues():
    """eigen keeps a positive eigenvalue below EPS as it is and replaces only zero or negative ones by EPS (checked against
    eigh by hand); an exactly singular C gives a finite C^{-1/2}, where flooring only D² < 0 would divide by zero."""
    r = np.random.default_rng(3)
    lam = np.array([1.0, 1e-3, 1e-9, 0.0, -1e-12])
    B, D = C.eigen(np.diag(lam))                                        # eigh is exact on a diagonal matrix
    np.testing.assert_array_equal(np.sort(D), np.sqrt([C.EPS, C.EPS, 1e-9, 1e-3, 1.0])[[2, 0, 1, 3, 4]])
    np.testing.assert_array_equal(np.abs(B), np.abs(B) @ np.eye(5))
    Q = np.linalg.qr(r.standard_normal((5, 5)))[0]                     # rotated: the same rule on eigh's eigenvalues
    A = Q @ np.diag(lam) @ Q.T
    B, D = C.eigen(A)
    ev = np.linalg.eigh((A + A.T) / 2)[0]
    np.testing.assert_array_equal(D, np.sqrt(np.where(ev <= 0, C.EPS, ev)))
    assert np.abs(D ** 2 - 1e-9).min() < 1e-14                          # kept, not raised to EPS
    np.testing.assert_allclose(B.T @ B, np.eye(5), atol=1e-14)
    # exact zero: diag(1, 0) has a zero eigenvalue that eigh returns exactly
    B, D = C.eigen(np.diag([1.0, 0.0]))
    assert np.all(np.isfinite(1.0 / D)) and sorted(D ** 2) == [C.EPS, 1.0]
    s = C.CmaState(np.zeros(2), 0.5, 6)
    s.C = np.diag([1.0, 0.0])
    z = r.standard_normal((6, 2))
    _, Y = C.ask(s, z)
    C.tell(s, Y, C.sphere(Y))
    assert np.all(np.isfinite(s.C)) and np.all(np.isfinite(s.p_sigma)) and np.isfinite(s.sigma)


def test_tell_ranks_in_numpy_order():
    """NaN ranks after +inf, -0 equals +0, ties go to the lower sample index: the same update as the finite values
    listed in that order."""
    z = np.random.default_rng(4).standard_normal((8, 3))
    f = np.array([np.nan, np.inf, -0.0, -np.inf, 0.0, np.copysign(np.nan, -1.0), 1.0, 1.0])
    order = [3, 2, 4, 6, 7, 1, 0, 5]
    s1, s2 = C.CmaState(np.zeros(3), 1.0, 8), C.CmaState(np.zeros(3), 1.0, 8)
    _, Y = C.ask(s1, z)
    C.tell(s1, Y, f)
    C.tell(s2, Y[order], np.arange(8.0))
    np.testing.assert_array_equal(s1.mean, s2.mean)
    np.testing.assert_array_equal(s1.C, s2.C)


def test_tell_h_sigma_override():
    s1, s2, s3 = (C.CmaState(np.zeros(4), 1.0, 8) for _ in range(3))
    z = np.random.default_rng(5).standard_normal((8, 4))
    _, Y = C.ask(s1, z)
    f = C.sphere(Y)
    C.tell(s1, Y, f)
    C.tell(s2, Y, f, h_sigma=1.0)
    C.tell(s3, Y, f, h_sigma=0.0)
    assert np.array_equal(s1.pc, s2.pc) or np.array_equal(s1.pc, s3.pc)
    assert np.array_equal(s3.pc, np.zeros(4)) and not np.array_equal(s2.pc, s3.pc)
    assert s2.sigma == s3.sigma and np.array_equal(s2.p_sigma, s3.p_sigma)


def test_objectives_have_their_minimum_inside_the_cube():
    for n in (2, 4, 10, 32):
        for name in C.OBJECTIVES:
            f, xs, H = C.objective(name, n, seed=n)
            assert np.all((0 < xs) & (xs < 1)) and f(xs[None])[0] == 0.0
            X = np.random.default_rng(n).uniform(0, 1, (64, n))
            assert np.all(f(X) > 0)
            if H is None:
                continue
            # quadratic: f(x* + h) = ½ hᵀHh exactly (up to rounding), H has the advertised spectrum
            h = X - xs
            np.testing.assert_allclose(f(X), 0.5 * np.einsum("ki,ij,kj->k", h, H, h), rtol=1e-10)
            ev = np.linalg.eigvalsh(H) / 2
            cond = {"sphere": 1.0, "ellipsoid1e3": 1e3, "ellipsoid1e6": 1e6, "cigar": 1e6, "discus": 1e6}[name]
            np.testing.assert_allclose(ev.max() / ev.min(), cond, rtol=1e-6)
            if name in ("cigar", "discus"):
                big = np.sum(ev > 1e3)
                assert big == (n - 1 if name == "cigar" else 1)
    f, xs, _ = C.objective("rosenbrock", 3)
    assert f((xs + 1e-3)[None])[0] > 0
