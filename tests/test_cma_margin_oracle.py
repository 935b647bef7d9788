"""CPU: the CMA-ES with Margin oracle (oracle/cma_margin_oracle.py) and the `cmaes` service's `with_margin` levels.

* The margin step on hand-built states: the edge case fires exactly when min(p_lo, p_up) < α and leaves the state alone
  one ulp away; the side case's redistribution worked by hand; a binary dimension that plain CMA-ES has fixed gets its
  crossing probability back to α.
* The invariant (edge: crossing probability ≥ α; side: each tail in [min(α/2, 1e-10), 0.5]) over long randomized runs.
* With no discrete dimension the oracle is `cma_oracle` bit for bit.
* Level mapping of `int` (with and without `step`) and `discrete`, and encoding at and beside every threshold, by the
  service's encoder and the oracle's.
* How often CMAwM and plain rounding reach the optimum of an integer ellipsoid over fixed seeds.
"""
import numpy as np
import pytest
from scipy.stats import norm

from kubeflow_b200.suggestion import cma_margin as SM
from kubeflow_b200.suggestion.internal import HyperParameter
from oracle import cma_margin_oracle as M
from oracle import cma_oracle as O


# ------------------------------------------------------------------------------------------------ hand-built steps
def test_edge_case_fires_exactly_below_alpha():
    dims = {0: np.array([0.0, 1.0])}                       # one threshold at 0.5
    m, sigma, c = np.array([0.8]), 0.1, np.array([1.0])
    p_cross = float(norm.cdf((0.5 - 0.8) / 0.1))
    assert M.tails(0.8, 0.1, 0.5, 0.5)[0] == pytest.approx(p_cross, rel=1e-14)
    at = M.tails(0.8, 0.1, 0.5, 0.5)[0]
    m1, A1, cases = M.margin_step(m, [1.0], sigma, c, dims, at)                # min == α: left alone
    assert cases == {0: "edge"} and m1[0] == 0.8 and A1[0] == 1.0
    m2, A2, cases = M.margin_step(m, [1.0], sigma, c, dims, np.nextafter(at, 1.0))   # one ulp above: moved
    assert cases == {0: "edge-moved"} and A2[0] == 1.0 and m2[0] == pytest.approx(0.8, rel=1e-12)   # to where it was, to rounding
    assert M.tails(m2[0], 0.1, 0.5, 0.5)[0] == pytest.approx(np.nextafter(at, 1.0), rel=1e-12)
    # the lower boundary interval moves up towards ℓ the same way
    m3, _, cases = M.margin_step(np.array([0.2]), [1.0], sigma, c, dims, 0.05)
    assert cases == {0: "edge-moved"} and m3[0] == pytest.approx(0.5 - 0.1 * norm.isf(0.05), rel=1e-14)


def test_side_case_fixed_point_and_floor_by_hand():
    dims = {0: np.array([0.0, 0.5, 1.0])}                  # thresholds 0.25, 0.75; m = 0.5 in the middle interval
    chi = norm.isf(0.01)
    s = 0.25 / chi                                         # both tails 0.01, above α/2: nothing to take, A stays 1
    m, A, cases = M.margin_step(np.array([0.5]), [1.0], 1.0, np.array([s * s]), dims, 1e-3)
    assert cases == {0: "side"} and m[0] == pytest.approx(0.5, rel=1e-15) and A[0] == pytest.approx(1.0, rel=1e-13)
    s = 0.25 / 6.5                                         # tails Φ(−6.5) ≈ 4e-11 < α/2: both floored to α/2
    m, A, _ = M.margin_step(np.array([0.5]), [1.0], 1.0, np.array([s * s]), dims, 1e-3)
    assert m[0] == pytest.approx(0.5, rel=1e-15)
    assert A[0] == pytest.approx(0.5 / (2 * norm.isf(5e-4) * s), rel=1e-13)


def test_side_case_redistribution_by_hand():
    dims = {0: np.array([0.0, 0.5, 1.0])}
    m0, s, alpha = 0.6, 0.1, 0.01
    p_lo, p_up = norm.cdf((0.25 - m0) / s), norm.cdf((m0 - 0.75) / s)      # 2.3e-4 and 0.067
    p_mid = 1 - p_lo - p_up
    h = alpha / 2
    lo, up = max(p_lo, h), max(p_up, h)                    # the lower tail is floored, the upper is not
    assert lo == h and up == p_up
    over = 1 - lo - up - p_mid                             # the floor's overshoot, taken from the upper tail only
    q_up = up + over * (up - h) / (lo + p_mid + up - 3 * h)
    assert over < 0 and q_up < p_up
    chi_lo, chi_up = norm.isf(h), norm.isf(q_up)
    want_A = 0.5 / ((chi_lo + chi_up) * s)
    want_m = (0.25 * chi_up + 0.75 * chi_lo) / (chi_lo + chi_up)
    m, A, cases = M.margin_step(np.array([m0]), [1.0], s, np.array([1.0]), dims, alpha)
    assert cases == {0: "side"}
    assert A[0] == pytest.approx(want_A, rel=1e-13) and m[0] == pytest.approx(want_m, rel=1e-13)
    got_lo, got_up = M.tails(m[0], s * A[0], 0.25, 0.75)
    assert got_lo == pytest.approx(h, rel=1e-12) and got_up == pytest.approx(q_up, rel=1e-12)


def test_binary_dimension_fixed_by_plain_cma_gets_alpha_back():
    dims = {0: np.array([0.0, 1.0])}
    m, sigma, c, alpha = np.array([0.9, 0.3]), 1e-3, np.array([1.0, 1.0]), 1.0 / (2 * 10)
    assert M.tails(0.9, sigma, 0.5, 0.5)[0] == 0.0                          # plain CMA-ES: Φ(−400), the level is frozen
    m1, A1, cases = M.margin_step(m, [1.0, 1.0], sigma, c, dims, alpha)
    assert cases == {0: "edge-moved"} and m1[1] == 0.3 and A1[0] == 1.0
    assert M.tails(m1[0], sigma, 0.5, 0.5)[0] == pytest.approx(alpha, rel=1e-12)
    assert not M.invariant_violations(m1, A1, sigma, c, dims, alpha, cases, m)


# ------------------------------------------------------------------------------------------------ runs
def _mixed_dims(D):
    """every other dimension discrete: 5-level table, binary, a long arithmetic range, an uneven discrete list"""
    kinds = [np.linspace(0, 1, 5), np.array([0.0, 1.0]), (0.0, 1.0 / 5000, 5001), np.array([0.0, 0.1, 0.15, 0.6, 1.0])]
    return {j: kinds[(j // 2) % len(kinds)] for j in range(0, D, 2)}


@pytest.mark.parametrize("D,lam,seed", [(6, 8, 0), (10, 10, 1), (16, 12, 2)])
def test_invariant_over_long_randomized_runs(D, lam, seed):
    r = np.random.default_rng(seed)
    dims = _mixed_dims(D)
    xs = M.encode(dims, r.uniform(0, 1, D))
    ms = M.MarginState(np.full(D, 0.5), 1.0 / 6.0, lam, dims)
    seen = set()
    for g in range(400):
        X, Y, _ = M.ask(ms, r.standard_normal((lam, D)))
        f = ((np.clip(X, 0, 1) - xs) ** 2 * (1 + np.arange(D))).sum(1)
        M.tell(ms, Y, f)
        s = ms.state
        bad = M.invariant_violations(s.mean, ms.A, s.sigma, np.diag(s.C), dims, ms.alpha, ms.last_cases, ms.mean_before)
        assert not bad, f"generation {g}: {bad}"
        seen.update(ms.last_cases.values())
        if s.sigma < 1e-12:
            break
    assert {"edge-moved", "side"} <= seen


def test_no_discrete_dimension_is_cma_oracle_bit_for_bit():
    D, lam = 7, 9
    r1, r2 = np.random.default_rng(4), np.random.default_rng(4)
    ms = M.MarginState(np.full(D, 0.5), 0.2, lam, {})
    ref = O.CmaState(np.full(D, 0.5), 0.2, lam)
    f = lambda X: O.rastrigin((X - 0.3) * 5)
    for _ in range(60):
        X, Y, _ = M.ask(ms, r1.standard_normal((lam, D)))
        Xr, Yr = O.ask(ref, r2.standard_normal((lam, D)))
        assert np.array_equal(X, Xr) and np.array_equal(Y, Yr)
        M.tell(ms, Y, f(X))
        O.tell(ref, Yr, f(Xr))
        for k in ("mean", "C", "p_sigma", "pc"):
            assert np.array_equal(getattr(ms.state, k), getattr(ref, k)), k
        assert ms.state.sigma == ref.sigma and np.array_equal(ms.A, np.ones(D))


# ------------------------------------------------------------------------------------------------ levels and encoding
def test_int_levels_without_and_with_step():
    L = SM.discrete_dims([HyperParameter.int("a", "1", "5")])[0]
    assert np.array_equal(L.cube, [0.0, 0.25, 0.5, 0.75, 1.0]) and [L.value(u) for u in L.cube] == ["1", "2", "3", "4", "5"]
    L = SM.discrete_dims([HyperParameter.int("a", "0", "10", "3")])[0]
    assert np.allclose(L.cube, [0.0, 0.3, 0.6, 0.9], rtol=0, atol=1e-15)
    assert [L.value(u) for u in L.cube] == ["0", "3", "6", "9"]
    L = SM.discrete_dims([HyperParameter.int("a", "-5", str(2 ** 31))])[0]                   # too long for a table
    assert isinstance(L.cube, tuple) and L.cube[2] == 2 ** 31 + 6
    assert L.value(0.0) == "-5" and L.value(1.0) == str(2 ** 31) and L.value(L.cube[1] * 7) == "2"


def test_discrete_levels_sorted_distinct():
    L = SM.discrete_dims([HyperParameter.double("x", "0", "1"), HyperParameter.discrete("d", ["1", "0.1", "10", "1.0"])])
    assert list(L) == [1]
    L = L[1]
    assert np.allclose(L.cube, [0.0, 0.9 / 9.9, 1.0]) and [L.value(u) for u in L.cube] == ["0.1", "1", "10"]


@pytest.mark.parametrize("bad", [HyperParameter.discrete("d", ["a", "b"]), HyperParameter.discrete("d", ["2", "2.0"]),
                                 HyperParameter.int("i", "0", "3", "5")])
def test_unusable_levels_are_refused(bad):
    with pytest.raises(SM.AlgorithmSettingsError, match=bad.name):
        SM.discrete_dims([bad])


@pytest.mark.parametrize("dim", [np.linspace(0, 1, 5), np.array([0.0, 1.0]), np.array([0.0, 0.1, 0.15, 0.6, 1.0]),
                                 (0.0, 1.0 / 5000, 5001), (0.0, 0.3, 4)])
def test_encoding_at_and_beside_every_threshold(dim):
    K = M.count(dim)
    ks = np.arange(K - 1) if K < 50 else np.r_[0:20, K // 2 - 10:K // 2 + 10, K - 21:K - 1]
    table = {0: dim}
    levels = {0: SM.Levels(dim)}
    for k in ks:
        t = float(M.threshold(dim, k))
        for x, want in ((t, k), (np.nextafter(t, -np.inf), k), (np.nextafter(t, np.inf), k + 1)):
            lv = float(M.level(dim, want))
            assert M.encode(table, np.array([x]))[0] == lv, (k, x)
            assert SM.encode(levels, np.array([x]))[0] == lv, (k, x)
    for x, want in ((-3.0, 0), (7.0, K - 1)):
        assert M.encode(table, np.array([x]))[0] == SM.encode(levels, np.array([x]))[0] == float(M.level(dim, want))


# ------------------------------------------------------------------------------------------------ integer optimum
SEEDS = range(8)


def integer_ellipsoid_runs(margin: bool, seeds=SEEDS, D=6, K=11, lam=10, gens=300):
    """Oracle runs on an integer ellipsoid with levels 0..K−1 in every dimension: the number of seeds whose best sample
    is the integer optimum.  margin=False is plain CMA-ES whose samples are rounded to the nearest level (the service
    without with_margin)."""
    dims = {j: np.linspace(0, 1, K) for j in range(D)}
    hits = 0
    for seed in seeds:
        r = np.random.default_rng(100 + seed)
        xs = r.integers(0, K, D)
        w = 10.0 ** (3 * np.arange(D) / (D - 1))
        ms = M.MarginState(np.full(D, 0.5), 1.0 / 6.0, lam, dims if margin else {})
        best = np.inf
        for _ in range(gens):
            X, Y, _ = M.ask(ms, r.standard_normal((lam, D)))
            U = np.round(np.clip(X, 0, 1) * (K - 1))       # with the margin X is already on a level: this only reads it
            f = ((U - xs) ** 2 * w).sum(1)
            best = min(best, f.min())
            if best == 0:
                break
            M.tell(ms, Y, f)
        hits += best == 0
    return hits


def test_margin_reaches_the_integer_optimum_more_often_than_rounding():
    with_margin, rounding = integer_ellipsoid_runs(True), integer_ellipsoid_runs(False)
    print(f"\nMEASURED integer ellipsoid hits over {len(SEEDS)} seeds: with_margin {with_margin}, rounding {rounding}")
    assert with_margin == len(SEEDS) and with_margin > rounding
