"""CPU oracle for Katib's ``multivariate-tpe`` algorithm: Optuna's ``TPESampler(multivariate=True)`` with its defaults on a
flat search space, as Katib's Optuna service calls it.

TEST INFRASTRUCTURE ONLY (same rule as gp_oracle.py).  PARITY UNPINNED: neither Optuna nor Katib's Optuna service is in the
reference tree or installable here, so this is a NumPy / SciPy FP64 restatement written from memory of Optuna 3.x
(``optuna/samplers/_tpe/sampler.py``, ``parzen_estimator.py``, ``_truncnorm.py``).  Every function names the Optuna function
it restates.  What pins it offline (tests/test_mvtpe_oracle.py): hand-worked numbers, SciPy (``truncnorm.logpdf``, ``quad``
and ``norm`` CDF differences for integer masses), and KS / chi-square / joint-quadrant tests of its sampler.  This file is the
contract of the GPU path (kubeflow_b200/csrc/mvtpe.cu).

Details recalled rather than read, in one place:

* [RECALL] Katib's Optuna service accepts ``n_startup_trials`` (default 10), ``n_ei_candidates`` (default 24) and
  ``random_state`` for ``multivariate-tpe``, and builds ``TPESampler(multivariate=True, ...)`` with everything else at
  Optuna's defaults: consider_prior=True, prior_weight=1.0, consider_magic_clip=True, consider_endpoints=False.
* [RECALL] Space mapping: DOUBLE → FloatDistribution(min, max); INT → IntDistribution(min, max) (Katib passes no step; here
  ``step`` is honoured, q = step or 1, and the upper bound is the last grid point, as IntDistribution adjusts it);
  CATEGORICAL / DISCRETE → CategoricalDistribution(list), observed as the category index.  MAXIMIZE negates the objective.
  Trials with a NaN objective are failed in Optuna and never told.
* [RECALL] ``default_gamma(n) = min(ceil(0.1·n), 25)``; the split takes the n_below best in a stable loss order and both groups
  are put back in told order (``_split_complete_trials`` sorts by trial number).
* [RECALL] ``default_weights(m)``: ones for m < 25, else linspace(1/m, 1, m − 25) followed by 25 ones; the prior's weight is
  appended and the weights are normalised.
* [RECALL] Multivariate sigma: 0.2 · max(m, 1)^(−1/(D + 4)) · (hi' − lo') for every observation of a group, D = number of
  parameters in the space; integers widen the range by q/2 on each side; the prior component is N((lo' + hi')/2, hi' − lo');
  the magic clip is [(hi' − lo') / min(100, 1 + m + 1), hi' − lo'].
* [RECALL] Categoricals: an observation's row is prior_weight / C everywhere plus 1 at the observed index, normalised; the
  prior's row is uniform.
* [RECALL] Density of a vector: logsumexp_k(log w_k + Σ_d log p_kd(x_d)); floats a normal truncated to [lo, hi], integers the
  normal mass of [x − q/2, x + q/2] over that of [lo', hi'], categories the row entry.  ``_log_gauss_mass`` works in the left
  tail by symmetry; across 0 Optuna writes log1p(−Φ(a) − Φ(−b)), which is the same quantity as log(½(erf(b/√2) + erf(−a/√2)))
  used here — that form does not cancel for the narrow bins of integers with many levels.
* [RECALL] Sampling: each candidate picks one component ∝ w_k, then draws every parameter from it: floats and integers by the
  truncated normal (integers on [lo', hi'], then ``clip(lo + round((v − lo)/q)·q, lo, hi)``), categories from row k.  The
  decision is ``samples[np.argmax(log l − log g)]``; a batch of k is k independent asks of one model.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.special import erf, log_ndtr

LF = 25                   # the ramp length of default_weights and the cap of default_gamma
PRIOR_WEIGHT = 1.0
LN_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)


def n_below(n: int) -> int:
    """optuna.samplers._tpe.sampler.default_gamma."""
    return min(int(math.ceil(0.1 * n)), LF)


def default_weights(m: int) -> np.ndarray:
    """optuna.samplers._tpe.sampler.default_weights."""
    if m == 0:
        return np.asarray([])
    if m < LF:
        return np.ones(m)
    ramp = np.linspace(1.0 / m, 1.0, num=m - LF)
    return np.concatenate([ramp, np.ones(LF)])


def split_trials(losses):
    """optuna.samplers._tpe.sampler._split_complete_trials for one objective: the n_below best in a stable loss order (NumPy's
    order for ±inf) are "below", the rest "above"; both index lists in told order."""
    losses = np.asarray(losses, dtype=np.float64)
    nb = n_below(len(losses))
    order = np.argsort(losses, kind="stable")
    return np.sort(order[:nb]), np.sort(order[nb:])


def bounds(p):
    """(lo, hi, lo', hi', q) of a float or integer parameter; integers end at their last grid point and widen by q/2."""
    if p[0] == "float":
        return float(p[1]), float(p[2]), float(p[1]), float(p[2]), None
    lo, q = float(p[1]), float(p[3])
    levels = int(math.floor((float(p[2]) - lo) / q)) + 1
    hi = lo + (levels - 1) * q
    return lo, hi, lo - 0.5 * q, hi + 0.5 * q, q


def levels(p) -> int:
    if p[0] == "cat":
        return int(p[1])
    lo, hi, _, _, q = bounds(p)
    return int(round((hi - lo) / q)) + 1


def sigma(p, m: int, D: int) -> float:
    """optuna.samplers._tpe.parzen_estimator._ParzenEstimator._calculate_numerical_distributions (multivariate): the shared
    sigma of a group's observations, magic-clipped (the prior's sigma, hi' − lo', is the clip's upper end)."""
    _, _, lo2, hi2, _ = bounds(p)
    r = hi2 - lo2
    s = 0.2 * max(m, 1) ** (-1.0 / (D + 4)) * r
    return float(np.clip(s, r / min(100.0, 1.0 + (m + 1)), r))


def log_gauss_mass(a, b):
    """optuna.samplers._tpe._truncnorm._log_gauss_mass: log of the N(0, 1) mass of [a, b], elementwise, a < b."""
    a, b = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64))
    a, b = a.copy(), b.copy()
    right = a > 0
    a[right], b[right] = -b[right], -a[right]
    out = np.empty(a.shape)
    left = b <= 0
    la, lb = log_ndtr(a[left]), log_ndtr(b[left])
    out[left] = lb + np.log(-np.expm1(la - lb))
    c = ~left
    out[c] = np.log(0.5 * (erf(b[c] / math.sqrt(2.0)) + erf(-a[c] / math.sqrt(2.0))))
    return out


def float_logpdf(x, mu, sg, lo, hi):
    """optuna.samplers._tpe._truncnorm.logpdf: N(mu, sg²) truncated to [lo, hi] (−inf outside)."""
    x, mu = np.asarray(x, dtype=np.float64), np.asarray(mu, dtype=np.float64)
    z = (x - mu) / sg
    out = -0.5 * z * z - LN_SQRT_2PI - math.log(sg) - log_gauss_mass((lo - mu) / sg, (hi - mu) / sg)
    return np.where((x >= lo) & (x <= hi), out, -np.inf)


def int_logpmf(x, mu, sg, p):
    """optuna.samplers._tpe.probability_distributions._BatchedDiscreteTruncNormDistributions' log pdf: the normal mass of
    [x − q/2, x + q/2] ∩ [lo', hi'] over that of [lo', hi']."""
    lo, hi, lo2, hi2, q = bounds(p)
    x, mu = np.asarray(x, dtype=np.float64), np.asarray(mu, dtype=np.float64)
    xl, xu = np.maximum(x - 0.5 * q, lo2), np.minimum(x + 0.5 * q, hi2)
    return log_gauss_mass((xl - mu) / sg, (xu - mu) / sg) - log_gauss_mass((lo2 - mu) / sg, (hi2 - mu) / sg)


def build_models(space, X, losses):
    """optuna.samplers._tpe.sampler.TPESampler._sample's two _ParzenEstimator(multivariate=True) models.  X: n × D in parameter
    units (integers on their grid, category indices), told order.  Returns dict(n_below, below, above); each group is
    dict(idx, w, sigma, mu, cat_rows): its trials in told order, the normalised weights (observations, then the prior), sigma
    per parameter (NaN for categoricals), the observations (m × D) and per categorical (match, other) row entries."""
    D = len(space)
    X = np.asarray(X, dtype=np.float64).reshape(-1, D)
    below, above = split_trials(losses)
    out = dict(n_below=len(below))
    for name, idx in (("below", below), ("above", above)):
        m = len(idx)
        w = np.append(default_weights(m), PRIOR_WEIGHT)
        w = w / w.sum()
        sg = np.full(D, np.nan)
        cat_rows = np.full((D, 2), np.nan)
        for d, p in enumerate(space):
            if p[0] == "cat":
                a = PRIOR_WEIGHT / p[1]
                cat_rows[d] = (a + 1.0) / (PRIOR_WEIGHT + 1.0), a / (PRIOR_WEIGHT + 1.0)
            else:
                sg[d] = sigma(p, m, D)
        out[name] = dict(idx=idx, w=w, sigma=sg, mu=X[idx], cat_rows=cat_rows)
    return out


def component_logpdf(space, group, cands):
    """log p_k(x) of every candidate under every component of a group (observations in told order, the prior last):
    (M × (m + 1)), without the weights."""
    cands = np.asarray(cands, dtype=np.float64).reshape(-1, len(space))
    mu, sg, m = group["mu"], group["sigma"], len(group["w"]) - 1
    out = np.zeros((len(cands), m + 1))
    for d, p in enumerate(space):
        x = cands[:, d][:, None]
        if p[0] == "cat":
            C = p[1]
            obs = (x == mu[:, d][None, :])
            out[:, :m] += np.log(np.where(obs, group["cat_rows"][d, 0], group["cat_rows"][d, 1]))
            out[:, m] += -math.log(C)
            continue
        lo, hi, lo2, hi2, q = bounds(p)
        pm, ps = 0.5 * (lo2 + hi2), hi2 - lo2
        if p[0] == "float":
            out[:, :m] += float_logpdf(x, mu[:, d][None, :], sg[d], lo, hi)
            out[:, m] += float_logpdf(x[:, 0], pm, ps, lo, hi)
        else:
            out[:, :m] += int_logpmf(x, mu[:, d][None, :], sg[d], p)
            out[:, m] += int_logpmf(x[:, 0], pm, ps, p)
    return out


def log_density(space, group, cands):
    """optuna.samplers._tpe.parzen_estimator._ParzenEstimator.log_pdf: logsumexp_k(log w_k + log p_k(x))."""
    t = component_logpdf(space, group, cands) + np.log(group["w"])[None, :]
    mx = t.max(axis=1)
    return np.log(np.exp(t - mx[:, None]).sum(axis=1)) + mx


def score(space, models, cands):
    """optuna.samplers._tpe.sampler.TPESampler._compute_acquisition_func: log l(x) − log g(x)."""
    return log_density(space, models["below"], cands) - log_density(space, models["above"], cands)


def round_int(p, v):
    """IntDistribution's rounding of a draw: clip(lo + round((v − lo)/q)·q, lo, hi)."""
    lo, hi, _, _, q = bounds(p)
    return np.clip(lo + np.round((np.asarray(v) - lo) / q) * q, lo, hi)


def draw(space, models, M: int, rng):
    """optuna.samplers._tpe.parzen_estimator._ParzenEstimator.sample on the below model: M candidate vectors (M × D)."""
    from scipy.stats import truncnorm
    g = models["below"]
    m = len(g["w"]) - 1
    k = rng.choice(m + 1, size=M, p=g["w"])
    out = np.empty((M, len(space)))
    prior = k == m
    for d, p in enumerate(space):
        if p[0] == "cat":
            C = p[1]
            rows = np.full((m + 1, C), 1.0 / C)
            if m:
                rows[:m] = g["cat_rows"][d, 1]
                rows[np.arange(m), g["mu"][:, d].astype(int)] = g["cat_rows"][d, 0]
            cum = np.cumsum(rows, axis=1)
            u = rng.random(M)
            out[:, d] = np.minimum((u[:, None] >= cum[k]).sum(axis=1), C - 1)
            continue
        lo, hi, lo2, hi2, q = bounds(p)
        mu = np.where(prior, 0.5 * (lo2 + hi2), g["mu"][np.minimum(k, max(m - 1, 0)), d] if m else 0.0)
        sg = np.where(prior, hi2 - lo2, g["sigma"][d])
        v = truncnorm.rvs((lo2 - mu) / sg, (hi2 - mu) / sg, loc=mu, scale=sg, random_state=rng)
        out[:, d] = v if p[0] == "float" else round_int(p, v)
    return out


def marginal_cdf(space, group, d, x):
    """CDF of parameter d's marginal under a group's mixture (floats; integers before rounding, on [lo', hi'])."""
    from scipy.stats import norm
    p = space[d]
    _, _, lo2, hi2, _ = bounds(p)
    m = len(group["w"]) - 1
    mus = np.append(group["mu"][:, d], 0.5 * (lo2 + hi2))
    sgs = np.append(np.full(m, group["sigma"][d]), hi2 - lo2)
    x = np.asarray(x, dtype=np.float64)[..., None]
    num = norm.cdf((x - mus) / sgs) - norm.cdf((lo2 - mus) / sgs)
    den = norm.cdf((hi2 - mus) / sgs) - norm.cdf((lo2 - mus) / sgs)
    return (group["w"] * num / den).sum(-1)


def int_pmf(space, group, d):
    """Probabilities of parameter d's grid points under a group's mixture (an integer's marginal)."""
    p = space[d]
    lo, hi, lo2, hi2, q = bounds(p)
    grid = lo + np.arange(levels(p)) * q
    edges = np.concatenate([[lo2], grid + 0.5 * q])
    edges[-1] = hi2
    c = marginal_cdf(space, group, d, edges)
    return np.diff(c)


def cat_pmf(space, group, d):
    """Probabilities of parameter d's categories under a group's mixture."""
    C = space[d][1]
    m = len(group["w"]) - 1
    pr = np.full(C, group["w"][m] / C)
    for k in range(m):
        pr += group["w"][k] * group["cat_rows"][d, 1]
        pr[int(group["mu"][k, d])] += group["w"][k] * (group["cat_rows"][d, 0] - group["cat_rows"][d, 1])
    return pr


def choose(space, models, cands):
    """The decision: cands (M × D) → (the candidate at np.argmax of the scores, its index)."""
    cands = np.asarray(cands, dtype=np.float64)
    i = int(np.argmax(score(space, models, cands)))
    return cands[i], i
