"""CPU: the separable CMA-ES oracle (oracle/sepcma_oracle.py).  Its strategy parameters against `decimal` evaluations of the
recalled formulas, a D = 2 first tell worked by hand, invariants over long randomised runs, each termination criterion on a
constructed state, and what the algorithm is for: on a separable ill-conditioned objective it needs fewer evaluations
than full CMA-ES, on a rotated one more."""
from decimal import Decimal, getcontext

import numpy as np
import pytest

from oracle import cma_oracle as O
from oracle import cma_restart_oracle as R
from oracle import sepcma_oracle as S

getcontext().prec = 50


def _decimal_params(n, lam):
    n, mu = Decimal(n), lam // 2
    wp = [(Decimal(lam + 1) / 2).ln() - Decimal(i).ln() for i in range(1, mu + 1)]
    s = sum(wp)
    w = [x / s for x in wp]
    mu_eff = 1 / sum(x * x for x in w)
    c_sigma = (mu_eff + 2) / (n + mu_eff + 5)
    d_sigma = 1 + 2 * max(Decimal(0), ((mu_eff - 1) / (n + 1)).sqrt() - 1) + c_sigma
    c1 = 2 / ((n + Decimal("1.3")) ** 2 + mu_eff)
    cmu = min(1 - c1 - Decimal("1e-8"), (n + 2) / 3 * (2 / mu_eff / (n + Decimal(2).sqrt()) ** 2
                                                       + (1 - 1 / mu_eff) * min(Decimal(1), (2 * mu_eff - 1) / ((n + 2) ** 2 + mu_eff))))
    chi_n = n.sqrt() * (1 - 1 / (4 * n) + 1 / (21 * n * n))
    return dict(weights=w, mu_eff=mu_eff, c_sigma=c_sigma, d_sigma=d_sigma, cc=4 / (n + 4), c1=c1, cmu=cmu, chi_n=chi_n)


@pytest.mark.parametrize("n,lam", [(2, 6), (10, 10), (1000, 24), (4096, 28), (128, 4096)])
def test_parameters_match_decimal(n, lam):
    p, want = S.SepParams(n, lam), _decimal_params(n, lam)
    assert p.mu == lam // 2 and len(p.weights) == p.mu and p.cm == 1.0
    w0 = want["weights"][0]
    for got, w in zip(p.weights, want["weights"]):
        assert abs(Decimal(got) - w) <= Decimal(2e-15) * w0      # ln((λ+1)/2) − ln i cancels for i near μ
    for k in ("mu_eff", "c_sigma", "d_sigma", "cc", "c1", "cmu", "chi_n"):
        assert abs(Decimal(getattr(p, k)) - want[k]) <= Decimal(8e-16) * abs(want[k]), k


def test_d2_first_tell_by_hand():
    lam = 6
    st = S.SepState([0.5, 0.5], 0.2, lam)
    p = st.p
    Y = np.array([[0.3, -1.0], [1.2, 0.4], [-0.5, 0.1], [2.0, 2.0], [0.0, -0.7], [-1.5, 0.9]])
    f = np.array([3.0, 0.5, 1.0, 9.0, 0.5, 4.0])       # rank: 1, 4 (tie → lower index), 2, 0, 5, 3
    best = [1, 4, 2]
    w = [float(x) for x in p.weights]
    yw = [sum(w[i] * Y[best[i]][j] for i in range(3)) for j in range(2)]
    S.tell(st, Y, f)
    assert np.allclose(st.mean, [0.5 + 0.2 * yw[0], 0.5 + 0.2 * yw[1]], rtol=0, atol=1e-15)
    k_s = np.sqrt(p.c_sigma * (2 - p.c_sigma) * p.mu_eff)
    ps = [k_s * yw[0], k_s * yw[1]]                      # d = 1 before the first tell
    assert np.allclose(st.p_sigma, ps, rtol=1e-15, atol=0)
    nps = np.hypot(*ps)
    assert st.sigma == pytest.approx(0.2 * np.exp(p.c_sigma / p.d_sigma * (nps / p.chi_n - 1)), rel=1e-15)
    h = 1.0 if nps / np.sqrt(1 - (1 - p.c_sigma) ** 2) < (1.4 + 2 / 3) * p.chi_n else 0.0
    k_c = np.sqrt(p.cc * (2 - p.cc) * p.mu_eff)
    pc = [h * k_c * yw[0], h * k_c * yw[1]]
    assert np.allclose(st.pc, pc, rtol=1e-15, atol=0)
    a = 1 + p.c1 * (1 - h) * p.cc * (2 - p.cc) - p.c1 - p.cmu
    C = [a + p.c1 * pc[j] ** 2 + p.cmu * sum(w[i] * Y[best[i]][j] ** 2 for i in range(3)) for j in range(2)]
    assert np.allclose(st.C, C, rtol=1e-15, atol=0)
    assert st.g == 1


@pytest.mark.parametrize("n,lam,name", [(1, 4, "sphere"), (3, 7, "ellipsoid1e6"), (20, 13, "rosenbrock"), (50, 100, "discus"),
                                        (10, 4096, "rastrigin")])
def test_invariants_over_long_randomised_runs(n, lam, name):
    f = (lambda X: O.rastrigin(X - 0.4)) if name == "rastrigin" else O.objective(name, n, seed=n)[0]
    r = np.random.default_rng(n)
    st = S.SepState(np.full(n, 0.5), 1 / 6, lam)
    assert abs(st.p.weights.sum() - 1.0) <= 1e-15 and (st.p.weights > 0).all()
    assert np.all(np.diff(st.p.weights) < 0)
    for _ in range(600):
        X, Y = S.ask(st, r.standard_normal((lam, n)))
        S.tell(st, Y, f(X) + 1e-3 * r.standard_normal(lam))
        assert np.all(st.C > 0) and np.isfinite(st.C).all() and 0 < st.sigma <= S.SIGMA_MAX
        assert np.isfinite(st.mean).all()


def test_d1_formulas():
    p = S.SepParams(1, 4)
    w1, w2 = np.log(2.5), np.log(2.5) - np.log(2)
    assert np.allclose(p.weights, [w1 / (w1 + w2), w2 / (w1 + w2)], rtol=1e-15)
    me = (w1 + w2) ** 2 / (w1 * w1 + w2 * w2)
    assert p.mu_eff == pytest.approx(me, rel=1e-15)
    assert p.cc == pytest.approx(0.8, rel=1e-15) and p.c1 == pytest.approx(2 / (2.3 ** 2 + me), rel=1e-15)
    assert p.cmu == pytest.approx(2 / me / (1 + np.sqrt(2)) ** 2 + (1 - 1 / me) * min(1, (2 * me - 1) / (9 + me)), rel=1e-15)
    assert p.chi_n == pytest.approx(1 - 1 / 4 + 1 / 21, rel=1e-15)


def test_rank_mu_rate_is_capped_at_large_populations():
    # the recalled formula gives about 5.0 here; uncapped, C's own coefficient 1 − c1 − cμ is negative and the run turns NaN
    p = S.SepParams(128, 4096)
    assert p.cmu == 1 - p.c1 - 1e-8
    assert S.SepParams(10, 10).cmu < 1 - S.SepParams(10, 10).c1 - 1e-8      # the default population is never capped


def test_zero_variance_is_floored_under_the_root():
    assert np.array_equal(S.sqrt_c([0.0, -1.0, 4.0]), [np.sqrt(O.EPS), np.sqrt(O.EPS), 2.0])


# ------------------------------------------------------------------------------------------------ termination test
def _stop(mean=(0.5, 0.5), sigma=0.1, C=(1.0, 1.0), pc=(0.1, 0.1), hist=None, g=1, term=20, tolx=1e-13):
    C = np.asarray(C, dtype=np.float64)
    hist = np.arange(2.0 * term) if hist is None else hist
    return S.should_stop(np.asarray(mean, dtype=np.float64), sigma, C, np.asarray(pc, dtype=np.float64), S.sqrt_c(C), hist, g, term, tolx)


def test_a_plain_state_sets_no_flag():
    assert _stop() == 0


def test_tolfun():
    assert _stop(hist=np.full(40, 2.5), g=21) == R.TOLFUN
    assert _stop(hist=np.full(40, 2.5), g=20) == 0                 # not before g > term
    h = np.full(40, 2.5)
    h[3] = np.nan
    assert _stop(hist=h, g=21) == 0


def test_tolx():
    assert _stop(sigma=1e-14, C=(1.0, 0.5), pc=(1.0, -3.0)) & R.TOLX
    assert not _stop(sigma=1e-14, C=(1.0, 20.0), pc=(1.0, 1.0)) & R.TOLX       # σ·C_j, not σ·√C_j
    assert not _stop(sigma=1e-14, C=(1.0, 1.0), pc=(1.0, 11.0)) & R.TOLX


def test_tolxup():
    assert _stop(sigma=2e4) & R.TOLXUP
    assert not _stop(sigma=2e4, C=(0.2, 0.2)) & R.TOLXUP


def test_noeffectcoord():
    assert _stop(mean=(1e17, 0.5), sigma=1.0) == R.NOEFFECTCOORD
    assert _stop(mean=(1e15, 0.5), sigma=1.0) == 0


def test_conditioncov():
    assert _stop(C=(1.0, 1e-29)) == R.CONDITIONCOV
    assert _stop(C=(1.0, 1e-27)) == 0


def test_no_noeffectaxis_bit():
    assert not _stop(mean=(1e17, 1e17), sigma=1.0) & R.NOEFFECTAXIS


def test_run_records_the_history_ring():
    run = S.Run(np.full(3, 0.5), 0.2, 7)
    r = np.random.default_rng(1)
    for g in range(run.term + 2):
        X, Y = S.ask(run.state, r.standard_normal((7, 3)))
        fl = run.tell(Y, np.full(7, 1.25))
    assert fl & R.TOLFUN and run.hist[0] == 1.25


# ------------------------------------------------------------------------------------------------ what it is for
def _ellipsoid(n, seed, rotated):
    r = np.random.default_rng(seed)
    xs = r.uniform(0.2, 0.8, n)
    Q = np.linalg.qr(r.standard_normal((n, n)))[0] if rotated else np.eye(n)
    s = 1e6 ** (np.arange(n) / (n - 1))
    return lambda X: ((((X - xs) @ Q.T) ** 2) * s).sum(1)


def _evaluations(kind, f, n, seed, budget):
    """Evaluations until a sample has f < 1e-8 from mean 0.5, σ = 1/6 at the default population, or None past budget."""
    lam = 4 + int(3 * np.log(n))
    r = np.random.default_rng(seed)
    st = S.SepState(np.full(n, 0.5), 1 / 6, lam) if kind == "sep" else O.CmaState(np.full(n, 0.5), 1 / 6, lam)
    ask, tell = (S.ask, S.tell) if kind == "sep" else (O.ask, O.tell)
    for g in range(budget // lam):
        X, Y = ask(st, r.standard_normal((lam, n)))
        fx = f(X)
        if fx.min() < 1e-8:
            return (g + 1) * lam
        tell(st, Y, fx)
    return None


def test_separable_ellipsoid_needs_fewer_evaluations_than_full_cma():
    n = 40
    f = _ellipsoid(n, 0, rotated=False)
    full = _evaluations("full", f, n, 0, 200_000)
    sep = _evaluations("sep", f, n, 0, 200_000)
    assert full is not None and sep is not None and sep < full, (sep, full)
    print(f"\nMEASURED separable 1e6 ellipsoid D=40: sep {sep} evaluations, full {full}")


def test_rotated_ellipsoid_needs_more_evaluations_than_full_cma():
    n = 40
    f = _ellipsoid(n, 0, rotated=True)
    full = _evaluations("full", f, n, 0, 200_000)
    assert full is not None
    sep = _evaluations("sep", f, n, 0, 2 * full)                 # sep-CMA cannot learn the rotation
    assert sep is None or sep > full, (sep, full)
    print(f"\nMEASURED rotated 1e6 ellipsoid D=40: full {full} evaluations, sep {'> ' + str(2 * full) if sep is None else sep}")
