"""CPU: the TPE restatement (oracle/tpe_oracle.py) against hand-worked mixtures and independent SciPy computations — the
pins of the contract the GPU path (tests/test_gpu_tpe.py) is held to."""
import numpy as np
import pytest
from scipy import integrate, stats
from scipy.special import logsumexp

from oracle import tpe_oracle as O


def _apn(mus, pw=1.0, pm=0.5, ps=1.0):
    return O.adaptive_parzen_normal(np.asarray(mus, dtype=float), pw, pm, ps)


def test_apn_no_and_one_observation():
    w, mu, sg = _apn([])
    assert w.tolist() == [1.0] and mu.tolist() == [0.5] and sg.tolist() == [1.0]
    w, mu, sg = _apn([0.2], pw=3.0)                     # prior_mu >= the observation: prior second
    assert mu.tolist() == [0.2, 0.5] and sg.tolist() == [0.5, 1.0] and np.allclose(w, [0.25, 0.75])
    w, mu, sg = _apn([0.7])                             # prior_mu < the observation: prior first
    assert mu.tolist() == [0.5, 0.7] and sg.tolist() == [1.0, 0.5] and np.allclose(w, [0.5, 0.5])
    w, mu, sg = _apn([0.5])                             # equal: prior second (hyperopt's strict <)
    assert mu.tolist() == [0.5, 0.5] and sg.tolist() == [0.5, 1.0]


def test_apn_two_observations_and_prior_positions():
    w, mu, sg = _apn([0.9, 0.1], pw=2.0)                # prior in the middle; min sigma = 1/4
    assert np.allclose(mu, [0.1, 0.5, 0.9]) and np.allclose(sg, [0.4, 1.0, 0.4]) and np.allclose(w, [0.25, 0.5, 0.25])
    w, mu, sg = _apn([0.8, 0.6])                        # prior at the lower end; gaps 0.1, 0.2 clipped up to 0.25
    assert np.allclose(mu, [0.5, 0.6, 0.8]) and np.allclose(sg, [1.0, 0.25, 0.25])
    w, mu, sg = _apn([0.3, 0.1])                        # prior at the upper end
    assert np.allclose(mu, [0.1, 0.3, 0.5]) and np.allclose(sg, [0.25, 0.25, 1.0])
    w, mu, sg = _apn([0.7, 0.5])                        # an observation equal to prior_mu: searchsorted puts the prior first
    assert np.allclose(mu, [0.5, 0.5, 0.7]) and np.allclose(sg, [1.0, 0.25, 0.25])


def test_apn_ties_and_all_equal():
    w, mu, sg = _apn([0.2, 0.2, 0.2])                   # zero gaps clip to ps / min(100, 1 + 4) = 0.2
    assert np.allclose(mu, [0.2, 0.2, 0.2, 0.5]) and np.allclose(sg, [0.2, 0.2, 0.3, 1.0])
    w, mu, sg = _apn([0.1, 0.3, 0.1, 0.3], pm=0.2)
    assert np.allclose(mu, [0.1, 0.1, 0.2, 0.3, 0.3]) and np.allclose(sg, [1 / 6, 1 / 6, 1.0, 1 / 6, 1 / 6])   # gaps 0, 0.1 < 1/6
    w, mu, sg = _apn(np.full(40, 0.9))                  # all equal, past the ramp: prior first, then one gap of 0.4, min sigma 1/42
    assert sg[0] == 1.0 and abs(sg[1] - 0.4) < 1e-15 and np.allclose(sg[2:], 1 / 42) and abs(w.sum() - 1) < 1e-15


@pytest.mark.parametrize("n", [25, 26, 27])
def test_linear_forgetting_starts_past_25(n):
    lf = O.linear_forgetting_weights(n)
    if n == 25:
        assert lf.tolist() == [1.0] * 25
    elif n == 26:
        assert np.allclose(lf, [1 / 26] + [1.0] * 25)
    else:
        assert np.allclose(lf, [1 / 27, 1.0] + [1.0] * 25)
    mus = np.linspace(0.9, 0.0, n)                      # told order = descending values: the oldest is the largest
    w, mu, sg = _apn(mus, pw=1.0, pm=0.5)
    top = np.argmax(mu)                                 # the oldest observation carries the first ramp weight
    assert np.isclose(w[top] / w[np.argmin(mu)], lf[0]) and np.isclose(w[mu == 0.5].sum() / w[np.argmin(mu)], 1.0)


def test_n_below_and_split():
    assert [O.n_below(n, 0.25) for n in (0, 1, 9, 16, 17, 10000, 10 ** 6)] == [0, 1, 1, 1, 2, 25, 25]
    losses = [3.0, np.nan, 1.0, 1.0, np.inf, -np.inf]
    below, above = O.ap_split_trials(losses, 0.9)       # n_below = ceil(0.9·√6) = 3: -inf, then the tied 1.0s in told order
    assert below.tolist() == [2, 3, 5] and above.tolist() == [0, 1, 4]
    below, _ = O.ap_split_trials([1.0, 1.0, 1.0, 0.5], 0.75)
    assert below.tolist() == [0, 3]


def _model(seed, n, lo=-2.0, hi=3.0):
    r = np.random.default_rng(seed)
    obs = r.uniform(lo, hi, n)
    w, mu, sg = O.adaptive_parzen_normal(obs, 1.0, 0.5 * (lo + hi), hi - lo)
    return w, mu, sg, lo, hi


@pytest.mark.parametrize("n", [0, 1, 5, 30])
def test_continuous_lpdf_against_scipy_truncnorm(n):
    w, mu, sg, lo, hi = _model(n, n)
    x = np.random.default_rng(99).uniform(lo, hi, 200)
    got = O.GMM1_lpdf(x, w, mu, sg, lo, hi)
    a, b = (lo - mu) / sg, (hi - mu) / sg
    mass = stats.norm.cdf(b) - stats.norm.cdf(a)
    pk = w * mass / (w * mass).sum()                    # component probabilities of the truncated mixture
    ref = logsumexp(np.log(pk) + stats.truncnorm.logpdf(x[:, None], a, b, loc=mu, scale=sg), axis=1)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("q", [1.0, 0.5])
def test_quantized_lpdf_against_quad(q):
    w, mu, sg, lo, hi = _model(7, 12, lo=0.0, hi=6.0)
    pa = (w * (stats.norm.cdf(hi, mu, sg) - stats.norm.cdf(lo, mu, sg))).sum()
    xs = np.arange(0.0, 6.0 + q / 2, q)
    got = O.GMM1_lpdf(xs, w, mu, sg, lo, hi, q=q)
    for x, g in zip(xs, got):
        a, b = max(x - q / 2, lo), min(x + q / 2, hi)
        val, _ = integrate.quad(lambda t: (w * stats.norm.pdf(t, mu, sg)).sum(), a, b, epsabs=1e-14, epsrel=1e-12)
        assert abs(g - np.log(val / pa)) < 1e-9


def test_sampler_ks_against_truncated_mixture():
    w, mu, sg, lo, hi = _model(3, 20)
    x = O.GMM1_raw(w, mu, sg, lo, hi, np.random.default_rng(2024), 50000)
    assert (x >= lo).all() and (x < hi).all()
    ks = stats.kstest(x, lambda t: O.truncated_mixture_cdf(t, w, mu, sg, lo, hi))
    assert ks.statistic < 1.95 / np.sqrt(len(x)), ks            # the 1e-3-level critical value
    assert np.array_equal(O.quantize([0.5, 1.5, 2.5, -0.5, 7.4], 1.0), [0.0, 2.0, 2.0, -0.0, 7.0])   # half to even
    assert np.allclose(O.quantize([3.0, 7.4, 12.6], 5.0), [5.0, 5.0, 15.0])


def test_categorical_tables_by_hand():
    np.testing.assert_allclose(O.ap_categorical_tables([0, 2, 2], 1.0, 3), np.array([2.0, 1.0, 3.0]) / 6)
    np.testing.assert_allclose(O.ap_categorical_tables([], 0.5, 4), np.full(4, 0.25))
    obs = [1] + [0] * 25                                 # 26 observations: the oldest weighs 1/26
    np.testing.assert_allclose(O.ap_categorical_tables(obs, 1.0, 2), np.array([26.0, 1 + 1 / 26]) / (27 + 1 / 26))


def test_choose_is_first_index_argmax_per_parameter():
    space = [("uniform", 0.0, 1.0), ("quniform", 0.0, 10.0, 1.0), ("choice", 3)]
    X = np.array([[0.1, 2, 0], [0.2, 3, 1], [0.9, 9, 2], [0.15, 2, 0]], dtype=float)
    models, nb = O.build_models(space, X, [0.1, 0.5, 0.9, 0.2], gamma=0.9)
    assert nb == 2
    cands = [np.array([0.12, 0.12, 0.95]), np.array([2.2, 1.8, 9.0]), np.array([0.0, 2.0, 0.0])]
    vals, idx = O.choose(models, cands)
    assert idx.tolist() == [0, 0, 0] and vals.tolist() == [0.12, 2.0, 0.0]      # duplicates and equal levels: first occurrence
