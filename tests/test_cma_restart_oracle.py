"""CPU: the CMA-ES restart oracle (oracle/cma_restart_oracle.py): each termination criterion on hand-built states and on
their neighbours one ulp or one generation away, NaN and inf in the fitness history, the IPOP and BIPOP schedules, and
seeded sphere runs that end by TOLFUN or TOLX."""
import numpy as np
import pytest

from oracle import cma_oracle as O
from oracle import cma_restart_oracle as R

N = 3


def _state(**kw):
    """A state on which no criterion holds: spread history, σ = 0.1, C = B = I, d = 1, p_c = 0.01, g = 5 < term."""
    s = dict(mean=np.full(N, 0.5), sigma=0.1, C=np.eye(N), pc=np.full(N, 0.01), B=np.eye(N), d=np.ones(N),
             hist=np.linspace(0.0, 1.0, 2 * 20), g=5, term=20, tol_x=R.tolx(1.0 / 6.0))
    s.update(kw)
    return s


def _flags(**kw):
    return R.should_stop(**_state(**kw))


def test_base_state_is_quiet():
    assert _flags() == 0


def test_tolfun_range_and_generation():
    h = np.zeros(40)
    assert _flags(hist=h, g=21) & R.TOLFUN
    assert not _flags(hist=h, g=20) & R.TOLFUN                          # g > term, strictly
    h[7] = R.TOL_FUN
    assert not _flags(hist=h, g=21) & R.TOLFUN                          # range == tolfun: not below it
    h[7] = np.nextafter(R.TOL_FUN, 0.0)
    assert _flags(hist=h, g=21) & R.TOLFUN


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_tolfun_nan_and_inf_in_history(bad):
    h = np.zeros(40)
    h[3] = bad
    assert not _flags(hist=h, g=21) & R.TOLFUN
    assert not _flags(hist=np.full(40, np.inf), g=21) & R.TOLFUN       # inf − inf is NaN
    assert not _flags(hist=np.full(40, -np.inf), g=21) & R.TOLFUN


def test_history_records_best_and_worst_in_numpy_order():
    h = np.zeros(8)
    R.record(h, 5, 4, [3.0, np.nan, -1.0, np.inf])
    assert h[2] == -1.0 and np.isnan(h[3])                              # slot 2·(5 mod 4); NaN sorts last
    R.record(h, 4, 4, [np.inf, -np.inf, 0.0, 1.0])
    assert h[0] == -np.inf and h[1] == np.inf


def test_tolx_threshold_and_signed_pc():
    tol = 1e-12
    c = np.diag(np.full(N, np.nextafter(tol, 0.0)))
    assert _flags(sigma=1.0, C=c, pc=np.zeros(N), tol_x=tol) & R.TOLX
    c2 = c.copy()
    c2[1, 1] = tol
    assert not _flags(sigma=1.0, C=c2, pc=np.zeros(N), tol_x=tol) & R.TOLX
    assert not _flags(sigma=1.0, C=c, pc=np.full(N, tol), tol_x=tol) & R.TOLX
    assert _flags(sigma=1.0, C=c, pc=np.full(N, -1.0), tol_x=tol) & R.TOLX   # p_c is compared signed, as recalled


def test_tolxup_threshold():
    d = np.ones(N)
    d[2] = R.TOL_XUP
    assert not _flags(sigma=1.0, d=d) & R.TOLXUP
    d[2] = np.nextafter(R.TOL_XUP, np.inf)
    assert _flags(sigma=1.0, d=d) & R.TOLXUP
    d[0] = np.nan
    assert not _flags(sigma=1.0, d=d) & R.TOLXUP                        # max with a NaN is NaN


def _largest(pred, lo, hi):
    """Bisection over positive floats: the largest x in [lo, hi) with pred(x) (pred(lo) holds, pred(hi) fails, pred
    monotone), and its successor, for which pred fails."""
    assert pred(lo) and not pred(hi)
    while np.nextafter(lo, np.inf) < hi:
        mid = np.sqrt(lo * hi) if hi / lo > 2 else lo + (hi - lo) / 2
        mid = min(max(mid, np.nextafter(lo, np.inf)), np.nextafter(hi, 0.0))
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo, hi


def test_noeffectcoord_one_ulp():
    m = np.full(N, 1.0)
    sig, up = _largest(lambda s: 1.0 == 1.0 + (0.2 * s) * 1.0, 1e-17, 1e-15)
    assert _flags(mean=m, sigma=sig) & R.NOEFFECTCOORD
    assert not _flags(mean=m, sigma=up) & R.NOEFFECTCOORD
    m2 = m.copy()
    m2[1] = 1e17                                                         # any coordinate suffices
    assert _flags(mean=m2, sigma=0.1) & R.NOEFFECTCOORD
    assert not _flags(mean=m, sigma=0.1) & R.NOEFFECTCOORD


def test_noeffectaxis_one_generation_and_one_ulp():
    m = np.full(N, 1.0)
    d = np.array([1.0, 2.0, 2.0])
    sig, up = _largest(lambda s: 1.0 == 1.0 + (0.1 * s) * 1.0, 1e-17, 1e-14)
    assert _flags(mean=m, sigma=sig, d=d, g=3) & R.NOEFFECTAXIS           # axis 3 mod 3 = 0
    assert not _flags(mean=m, sigma=sig, d=d, g=4) & R.NOEFFECTAXIS       # axis 1: twice the step
    assert not _flags(mean=m, sigma=up, d=d, g=3) & R.NOEFFECTAXIS
    Q = np.linalg.qr(np.random.default_rng(0).standard_normal((N, N)))[0]
    assert not _flags(mean=m, sigma=sig * 0.5, B=Q, d=np.full(N, 4.0), g=3) & R.NOEFFECTAXIS
    assert _flags(mean=m, sigma=sig * 0.1, B=Q, d=np.full(N, 1.0), g=3) & R.NOEFFECTAXIS


def test_conditioncov_one_ulp():
    lo = 1e-7
    hi, up = _largest(lambda x: not x / lo > R.TOL_CONDITIONCOV, 1.0, 1e8)
    assert not _flags(d=np.array([lo, 1.0, hi])) & R.CONDITIONCOV
    assert _flags(d=np.array([lo, 1.0, up])) & R.CONDITIONCOV
    assert _flags(d=np.array([lo, 1.0, np.inf])) & R.CONDITIONCOV         # inf / finite
    assert not _flags(d=np.array([np.inf, np.inf, np.inf])) & R.CONDITIONCOV
    assert not _flags(d=np.array([lo, np.nan, up])) & R.CONDITIONCOV


def test_term_and_tolx_constants():
    assert R.funhist_term(10, 10) == 40 and R.funhist_term(128, 4096) == 11 and R.funhist_term(128, 4) == 970
    assert R.funhist_term(2, 6) == 20 and R.tolx(0.5) == 0.5e-12


def test_ipop_sequence_reaches_the_cap():
    s = R.Schedule("ipop", 128, sigma0=0.3, random_state=4)
    assert s.lam0 == 18
    lams = [s.next_run(0, 0)[0] for _ in range(11)]
    assert lams == [36, 72, 144, 288, 576, 1152, 2304, 4608, 8192, 8192, 8192]   # 18·2^9 = 9216 is the first capped
    assert all(h[2] == 0.3 for h in s.history)


def test_bipop_hand_worked_sequence():
    s = R.Schedule("bipop", 4, popsize0=10, sigma0=0.2)
    m = np.full(4, 0.5)
    # run 0: large, λ 10, 50 generations → budgets (small 0, large 500): small, λ_l = 10
    lam, _, sig = s.next_run(10, 50, draws=(m, (0.5, 0.25)))
    assert (s.regime, lam) == ("small", 8) and sig == pytest.approx(0.2 * 10 ** -0.5, rel=1e-15)   # ⌊10·0.5^0.25⌋ = 8
    # run 1: small λ 8 × 20 → (160, 500): small again, ⌊10·0.5^1⌋ = 5, σ0·10^0
    lam, _, sig = s.next_run(8, 20, draws=(m, (1.0, 0.0)))
    assert (s.regime, lam, sig) == ("small", 5, 0.2)
    # run 2: small λ 5 × 100 → (660, 500): large, i = 1, λ 20, σ0
    lam, _, sig = s.next_run(5, 100, draws=(m, (0.9, 0.9)))
    assert (s.regime, lam, sig) == ("large", 20, 0.2)
    # run 3: large λ 20 × 30 → (660, 1100): small, ⌊10·(½·20/10)^{U1²}⌋ = 10, σ0·10^{−1}
    lam, _, sig = s.next_run(20, 30, draws=(m, (0.3, 0.5)))
    assert (s.regime, lam) == ("small", 10) and sig == pytest.approx(0.02, rel=1e-15)
    # run 4: small λ 10 × 50 → (1160, 1100): large, i = 2, λ 40
    lam, _, sig = s.next_run(10, 50, draws=(m, (0.1, 0.1)))
    assert (s.regime, lam, sig) == ("large", 40, 0.2)
    assert s.budget == {"small": 1160, "large": 1100}


def test_bipop_small_runs_stay_at_least_four():
    s = R.Schedule("bipop", 2, sigma0=0.2)
    assert s.lam0 == 6
    lam, _, _ = s.next_run(6, 10, draws=(np.zeros(2), (1.0, 0.0)))      # ⌊6·0.5⌋ = 3 → clamped
    assert lam == 4


def test_restart_draws_are_seeded_by_state_and_index():
    a, ua = R.restart_draws(3, 1, 5, True)
    b, ub = R.restart_draws(3, 1, 5, True)
    c, _ = R.restart_draws(3, 2, 5, True)
    m, u = R.restart_draws(3, 1, 5, False)
    assert np.array_equal(a, b) and np.array_equal(ua, ub) and not np.array_equal(a, c)
    assert np.array_equal(a, m) and u is None                           # the mean is drawn first either way
    assert ((a >= 0) & (a < 1)).all() and ((ua >= 0) & (ua < 1)).all()


@pytest.mark.parametrize("D", [2, 10])
def test_seeded_sphere_run_stops_by_tolfun_or_tolx(D):
    lam = R.default_popsize(D)
    run = R.Run(np.full(D, 0.5), 1.0 / 6.0, lam)
    r = np.random.default_rng(D)
    xs = np.linspace(0.2, 0.7, D)
    for g in range(1, 3000):
        X, Y = O.ask(run.state, r.standard_normal((lam, D)))
        flags = run.tell(Y, O.sphere(X - xs))
        if flags:
            break
    assert flags & (R.TOLFUN | R.TOLX), (g, flags)
    assert not flags & (R.TOLXUP | R.CONDITIONCOV)
    assert np.linalg.norm(run.state.mean - xs) < 1e-4
