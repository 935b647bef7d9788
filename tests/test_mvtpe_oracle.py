"""CPU: oracle/mvtpe_oracle.py (the contract of ``multivariate-tpe``) against hand-worked numbers and SciPy, and its sampler by
KS, chi-square and a joint check that independent marginals fail."""
import math

import numpy as np
import pytest
from scipy import integrate, stats

from oracle import mvtpe_oracle as O


@pytest.mark.parametrize("n,nb", [(0, 0), (1, 1), (9, 1), (10, 1), (11, 2), (30, 3), (31, 4), (249, 25), (250, 25), (251, 25)])
def test_gamma_break_points(n, nb):
    assert O.n_below(n) == nb                     # min(ceil(0.1 n), 25)


@pytest.mark.parametrize("m", [0, 1, 24, 25, 26, 27, 100])
def test_weight_tables(m):
    w = O.default_weights(m)
    assert len(w) == m
    if m <= 25:
        assert (w == 1.0).all()
    else:
        ramp = w[: m - 25]
        assert ramp[0] == 1.0 / m and ramp[-1] == 1.0 if m - 25 > 1 else ramp[0] == 1.0 / m
        assert (w[m - 25:] == 1.0).all() and (np.diff(ramp) > 0).all()
    # a group of m observations: the prior's weight 1 appended, then normalised (m + 25 trials put m in the above group
    # whenever 0.1·(m + 25) >= 25, i.e. from m = 225; below that, pick n so that the above group has m)
    n = next(n for n in range(m, m + 26) if n - O.n_below(n) == m)
    g = O.build_models([("float", 0.0, 1.0)], np.zeros((n, 1)), np.arange(n, dtype=float))["above"]
    assert len(g["w"]) == m + 1 and g["w"][-1] == pytest.approx(1.0 / (w.sum() + 1.0), rel=1e-15)
    assert g["w"][:m] == pytest.approx(w / (w.sum() + 1.0), rel=1e-15)


def test_sigma_and_clip_by_hand():
    # float [0, 10], m = 16, D = 4: 0.2 · 16^(-1/8) · 10 = 2 / sqrt(2) = 1.41421...
    assert O.sigma(("float", 0.0, 10.0), 16, 4) == pytest.approx(2.0 / math.sqrt(2.0), rel=1e-15)
    # integer 0..9 step 1 widens to [-0.5, 9.5]: range 10; m = 0 uses max(m, 1) = 1: 0.2 · 10 = 2, below the clip's 10 / 2
    assert O.sigma(("int", 0, 9, 1), 0, 4) == pytest.approx(5.0, rel=1e-15)
    # m = 40, D = 0: 0.2 · 40^(-1/4) · 10 = 0.7953; lower end 10 / 42 = 0.238
    assert O.sigma(("int", 0, 9, 1), 40, 0) == pytest.approx(2.0 * 40 ** -0.25, rel=1e-15)
    # the clip's lower end: range / min(100, m + 2); m = 10^9, D = 0: 0.2 · 10^(-9/4) · 10 = 0.0112 < 10 / 100
    assert O.sigma(("float", 0.0, 10.0), 10 ** 9, 0) == pytest.approx(0.1, rel=1e-15)
    assert O.sigma(("float", 0.0, 10.0), 10 ** 6, 1) == pytest.approx(2.0 * 10 ** -1.2, rel=1e-14)
    # m = 3: lower end 10 / 5 = 2 > 0.2 · 3^(-1/5) · 10 = 1.60
    assert O.sigma(("float", 0.0, 10.0), 3, 1) == pytest.approx(2.0, rel=1e-15)
    # step 3 on [1, 12]: grid 1, 4, 7, 10 (hi is the last grid point), widened to [-0.5, 11.5]
    assert O.bounds(("int", 1, 12, 3)) == (1.0, 10.0, -0.5, 11.5, 3.0) and O.levels(("int", 1, 12, 3)) == 4


@pytest.mark.parametrize("mu,sg", [(0.3, 0.05), (-2.0, 0.7), (5.0, 0.01), (1.0, 30.0)])
def test_float_logpdf_against_scipy_truncnorm(mu, sg):
    lo, hi = -1.0, 3.0
    x = np.linspace(lo, hi, 41)
    ref = stats.truncnorm.logpdf(x, (lo - mu) / sg, (hi - mu) / sg, loc=mu, scale=sg)
    got = O.float_logpdf(x, mu, sg, lo, hi)
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("mu,sg", [(3.0, 0.8), (0.0, 2.5), (9.0, 0.2)])
def test_int_masses_against_quad_and_cdf_differences(mu, sg):
    p = ("int", 0, 9, 1)
    lo, hi, lo2, hi2, q = O.bounds(p)
    x = np.arange(10.0)
    got = np.exp(O.int_logpmf(x, mu, sg, p))
    Z = integrate.quad(lambda t: stats.norm.pdf(t, mu, sg), lo2, hi2, epsabs=0, epsrel=1e-13)[0]
    ref_q = np.array([integrate.quad(lambda t: stats.norm.pdf(t, mu, sg), v - 0.5, v + 0.5, epsabs=0, epsrel=1e-13)[0] for v in x]) / Z
    ref_c = (stats.norm.cdf(x + 0.5, mu, sg) - stats.norm.cdf(x - 0.5, mu, sg)) / (stats.norm.cdf(hi2, mu, sg) - stats.norm.cdf(lo2, mu, sg))
    big = ref_q > 1e-200
    np.testing.assert_allclose(got[big], ref_q[big], rtol=1e-9)
    np.testing.assert_allclose(got[ref_c > 1e-6], ref_c[ref_c > 1e-6], rtol=1e-9)     # the CDF difference cancels below that
    assert abs(got.sum() - 1.0) < 1e-12


def _mp_log_mass(a, b):
    import mpmath
    with mpmath.workdps(60):
        cdf = lambda x: mpmath.ncdf(mpmath.mpf(x))
        return float(mpmath.log(cdf(b) - cdf(a)))


def test_gauss_mass_far_tails_where_the_naive_difference_is_zero():
    """Against 60-digit values: intervals far in either tail, where Φ(b) − Φ(a) is 0 in FP64, and wide or central ones."""
    for a, b in ((40.0, 40.5), (200.0, 201.0)):
        assert stats.norm.cdf(b) - stats.norm.cdf(a) == 0.0
    for a, b in ((40.0, 40.5), (-40.5, -40.0), (-1e3, -999.0), (200.0, 201.0), (8.0, 9.0), (-37.5, -6.0), (-2.0, 3.0), (-0.5, 0.5)):
        lg = float(O.log_gauss_mass(a, b))
        ref = _mp_log_mass(a, b)
        assert abs(lg - ref) <= 1e-14 * abs(ref) + 1e-15, (a, b, lg, ref)
    # narrow bins: across 0 the erf sum keeps full precision; in a tail the difference of two log Φ loses ~1e-16·|log Φ| / width
    for a, b, tol in ((-1e-7, 1e-7, 1e-14), (-1e-7, 3e-7, 1e-14), (3.0, 3.0 + 1e-9, 1e-6), (-30.0, -30.0 + 1e-6, 1e-8)):
        ref = _mp_log_mass(a, b)
        assert abs(float(O.log_gauss_mass(a, b)) - ref) <= tol * abs(ref), (a, b)


def test_hand_evaluated_two_component_mixture():
    """2-D float space, one observation per group: below = {(0.2, 0.8)} (loss 0), above = {(0.9, 0.1)} (loss 1)."""
    space = [("float", 0.0, 1.0), ("float", 0.0, 1.0)]
    X = np.array([[0.2, 0.8], [0.9, 0.1]])
    md = O.build_models(space, X, [0.0, 1.0])
    b = md["below"]
    s = 0.2 * 1.0 ** (-1 / 6) * 1.0                          # m = 1, D = 2
    assert b["sigma"][0] == pytest.approx(max(s, 1 / 3), rel=1e-15)   # the clip: 1 / min(100, 3)
    s = 1 / 3
    assert b["w"].tolist() == [0.5, 0.5]
    x = np.array([[0.3, 0.7]])
    Zo = lambda mu: stats.norm.cdf((1 - mu) / s) - stats.norm.cdf((0 - mu) / s)
    po = stats.norm.pdf(0.3, 0.2, s) / Zo(0.2) * stats.norm.pdf(0.7, 0.8, s) / Zo(0.8)
    Zp = stats.norm.cdf(0.5) - stats.norm.cdf(-0.5)
    pp = (stats.norm.pdf(0.3, 0.5, 1.0) / Zp) * (stats.norm.pdf(0.7, 0.5, 1.0) / Zp)
    assert O.log_density(space, b, x)[0] == pytest.approx(math.log(0.5 * po + 0.5 * pp), rel=1e-12)
    a = md["above"]
    pa = stats.norm.pdf(0.3, 0.9, s) / Zo(0.9) * stats.norm.pdf(0.7, 0.1, s) / Zo(0.1)
    assert O.score(space, md, x)[0] == pytest.approx(math.log(0.5 * po + 0.5 * pp) - math.log(0.5 * pa + 0.5 * pp), rel=1e-12)


def test_categorical_rows_and_mixed_density():
    space = [("cat", 4), ("int", 0, 4, 2)]
    X = np.array([[2, 4], [0, 0]], dtype=float)
    md = O.build_models(space, X, [0.0, 1.0])
    b = md["below"]
    assert b["cat_rows"][0].tolist() == pytest.approx([1.25 / 2, 0.25 / 2])
    pm = np.exp(O.component_logpdf(space, b, np.array([[2, 4], [1, 2]])))
    assert pm[0, 0] == pytest.approx(1.25 / 2 * np.exp(O.int_logpmf(4.0, 4.0, b["sigma"][1], space[1])))
    assert pm[1, 1] == pytest.approx(0.25 * np.exp(O.int_logpmf(2.0, 2.0, 6.0, space[1])))
    tot = sum(np.exp(O.log_density(space, b, np.array([[c, v]]))[0]) for c in range(4) for v in (0, 2, 4))
    assert tot == pytest.approx(1.0, rel=1e-12)


def _models_for_sampler():
    space = [("float", -1.0, 3.0), ("int", 0, 19, 1), ("cat", 5), ("float", 0.0, 1.0)]
    r = np.random.default_rng(4)
    X = np.c_[r.uniform(-1, 3, 300), r.integers(0, 20, 300), r.integers(0, 5, 300), r.random(300)]
    return space, O.build_models(space, X, r.random(300))


def test_sampler_marginals_ks_and_chi_square():
    space, md = _models_for_sampler()
    M = 200_000
    C = O.draw(space, md, M, np.random.default_rng(11))
    g = md["below"]
    for d in (0, 3):
        ks = stats.kstest(C[:, d], lambda x: O.marginal_cdf(space, g, d, x))
        assert ks.pvalue > 1e-3, ks
    for d, pmf in ((1, O.int_pmf(space, g, 1)), (2, O.cat_pmf(space, g, 2))):
        cnt = np.bincount(C[:, d].astype(int), minlength=len(pmf))
        assert stats.chisquare(cnt, pmf * M).pvalue > 1e-3
    assert set(np.unique(C[:, 1])) <= set(range(20)) and set(np.unique(C[:, 2])) <= set(range(5))


def test_sampler_is_joint():
    """Two well-separated below observations at (0.1, 0.1) and (0.9, 0.9): every observation component puts its mass in its own
    quadrant, so the off-diagonal quadrants hold little beyond the prior's share.  Independent marginals would put half there."""
    space = [("float", 0.0, 1.0), ("float", 0.0, 1.0)]
    X = np.array([[0.1, 0.1], [0.9, 0.9]] + [[0.5, 0.5]] * 18)
    losses = np.array([0.0, 0.0] + [1.0] * 18)
    md = O.build_models(space, X, losses)
    assert md["n_below"] == 2
    C = O.draw(space, md, 100_000, np.random.default_rng(3))
    off = ((C[:, 0] < 0.5) != (C[:, 1] < 0.5)).mean()
    # sigma = 0.25 (the clip: 1 / 4); an observation component keeps P = (Φ(1.6) - Φ(-0.4)) / (Φ(3.6) - Φ(-0.4)) on its own
    # side in each coordinate; the prior (weight 1/3) puts half its mass off the diagonal
    P = (stats.norm.cdf(1.6) - stats.norm.cdf(-0.4)) / (stats.norm.cdf(3.6) - stats.norm.cdf(-0.4))
    expect = 2 / 3 * 2 * P * (1 - P) + 1 / 3 * 0.5
    assert abs(off - expect) < 0.01 and off < 0.3
    prod = np.mean(C[:, 0] < 0.5) * np.mean(C[:, 1] >= 0.5) + np.mean(C[:, 0] >= 0.5) * np.mean(C[:, 1] < 0.5)
    assert prod > 0.45                             # what independent marginals with the same laws would give


def test_choose_is_first_index_of_the_maximum():
    space, md = _models_for_sampler()
    C = O.draw(space, md, 512, np.random.default_rng(5))
    C = np.concatenate([C, C])
    x, i = O.choose(space, md, C)
    s = O.score(space, md, C)
    assert i == int(np.argmax(s)) and i < 512 and (x == C[i]).all()


@pytest.mark.parametrize("big", [False, True])
def test_torch_restatement_matches_the_oracle(big):
    """tests/_mvtpe_ref.py (the GPU tests' exhaustive yardstick) against the NumPy oracle, on the CPU device.  An integer with
    2^18 levels has bins of width ~1e-4 σ: in a tail their log mass is a difference of two log Φ values whose last-bit
    differences between SciPy's and torch's log_ndtr are amplified by 1 / width, hence the looser tolerance there."""
    import torch
    from tests import _mvtpe_ref as R
    space = [("float", -1.0, 3.0), ("int", 0, 19, 1), ("cat", 5), ("float", 0.0, 1.0)] + ([("int", 0, (1 << 18) - 1, 1)] if big else [])
    r = np.random.default_rng(9)
    X = np.c_[r.uniform(-1, 3, 400), r.integers(0, 20, 400), r.integers(0, 5, 400), r.random(400)]
    if big:
        X = np.c_[X, r.integers(0, 1 << 18, 400)]
    md = O.build_models(space, X, r.random(400))
    C = O.draw(space, md, 3000, r)
    C[:5] = X[:5]
    C[5, 0], C[6, 0], C[7, 1], C[8, 3] = -1.0, 3.0, 19.0, 1.0
    ref = O.score(space, md, C)
    got = R.score(space, md, torch.tensor(C), chunk=512).numpy()
    np.testing.assert_allclose(got, ref, rtol=0, atol=(1e-9 if big else 1e-11) * (1 + np.abs(ref).max()))


@pytest.mark.parametrize("big", [False, True])
def test_tolerance_covers_the_restatement_against_the_oracle(big):
    """_mvtpe_ref.tol, the distance two correct FP64 evaluations of a score can lie apart, covers this restatement against the
    NumPy oracle for every candidate: mixed spaces of 4 and 5 parameters (the second with a 2^18-level integer, whose tail
    bins are the worst conditioned) and a 40-float space, with candidates at observations and on the bounds.  It is no more
    than 1e-8 anywhere, so a pick check under it still tells scores apart."""
    import torch
    from tests import _mvtpe_ref as R
    r = np.random.default_rng(19)
    for space in ([("float", -1.0, 3.0), ("int", 0, 19, 1), ("cat", 5), ("float", 0.0, 1.0)] + ([("int", 0, (1 << 18) - 1, 1)] if big else []),
                  [("float", 0.0, 1e-3), ("float", -1e6, 1e6), ("int", 3, 48, 5), ("cat", 64)] * (10 if big else 1)):
        X = np.stack([O.round_int(p, r.uniform(p[1], p[2], 400)) if p[0] == "int" else
                      r.integers(0, p[1], 400).astype(float) if p[0] == "cat" else r.uniform(p[1], p[2], 400) for p in space], axis=1)
        md = O.build_models(space, X, r.random(400))
        C = O.draw(space, md, 2000, r)
        C[:5] = X[:5]
        for d, p in enumerate(space[:4]):
            C[5 + d, d] = p[1] if p[0] != "cat" else p[1] - 1
        ref = O.score(space, md, C)
        s, T = R.score_tol(space, md, torch.tensor(C), chunk=512)
        err, T = np.abs(s.numpy() - ref), T.numpy()
        assert (err <= T).all(), (len(space), float(np.max(err / T)))
        assert T.max() < 1e-8 and np.array_equal(T, R.tol(space, md, torch.tensor(C), chunk=512).numpy())


def test_pick_check_accepts_ties_and_rejects_gaps():
    """_mvtpe_ref.pick_ok: within the tolerances a pick may be any candidate, at its first occurrence; past them only the
    first occurrence of the maximum."""
    import torch
    from tests import _mvtpe_ref as R
    C = torch.tensor([[0.0, 1.0], [1.0, 0.0], [2.0, 0.0], [3.0, 3.0], [1.0, 0.0]], dtype=torch.float64)
    T = torch.full((5,), 1e-10, dtype=torch.float64)
    tie = torch.tensor([0.0, 1.0, 1.0 + 1.5e-10, 0.5, 1.0], dtype=torch.float64)      # 1 and 2 closer than T1 + T2
    assert R.pick_ok(C, tie, T, 2)[0] and R.pick_ok(C, tie, T, 1)[0]
    ok, _, keys = R.pick_ok(C, tie, T, 4)                             # a copy of 1 after its first occurrence
    assert not ok and keys == 2
    assert not R.pick_ok(C, tie, T, 3)[0] and not R.pick_ok(C, tie, T, 0)[0]
    gap = torch.tensor([0.0, 1.0, 1.0 + 2.5e-10, 0.5, 1.0], dtype=torch.float64)      # 2 wins by more than T1 + T2
    assert R.pick_ok(C, gap, T, 2)[0] and not R.pick_ok(C, gap, T, 1)[0]
    dup = torch.tensor([0.0, 1.0, 0.5, 0.5, 1.0], dtype=torch.float64)               # the best twice: the first copy
    ok, _, keys = R.pick_ok(C, dup, T, 1)
    assert ok and keys == 1 and not R.pick_ok(C, dup, T, 4)[0]
