"""CPU oracle for Katib's ``tpe`` algorithm: hyperopt's ``tpe.suggest`` on a flat search space, as Katib's hyperopt service
calls it.

TEST INFRASTRUCTURE ONLY (same rule as gp_oracle.py).  PARITY UNPINNED: neither hyperopt nor Katib's hyperopt service is in
/root/reference or installable here, so this is a NumPy FP64 restatement written from memory of hyperopt 0.2's ``tpe.py``.
Every function names the hyperopt function it restates; details recalled rather than read are marked [RECALL].  What pins it
offline (tests/test_tpe_oracle.py): hand-worked mixtures, the densities against SciPy (``truncnorm`` + ``logsumexp``, ``quad``
over a quantization bin), the rejection sampler's KS statistic against the truncated-mixture CDF.  This file is the contract of
the GPU path (kubeflow_b200/csrc/tpe.cu).

Space: a list of ``("uniform", lo, hi)`` (Katib DOUBLE), ``("quniform", lo, hi, q)`` (INT, q = step or 1) or
``("choice", n_categories)`` (CATEGORICAL / DISCRETE; observations are category indices) [RECALL: Katib's mapping].

Two choices this restatement pins where hyperopt leaves the order of equal keys to NumPy's default (unstable) sort: the losses
and each parameter's observations are sorted stably (``kind="mergesort"``), so equal losses split by told order and equal
values keep told order (which matters only when linear forgetting gives them different weights).
"""
from __future__ import annotations

import numpy as np
from scipy.special import erf

LF = 25           # hyperopt.tpe.DEFAULT_LF
EPS = 1e-12       # hyperopt.tpe.EPS


def linear_forgetting_weights(N: int, LF: int = LF) -> np.ndarray:
    """hyperopt.tpe.linear_forgetting_weights: ones for N < LF, else a ramp linspace(1/N, 1, N - LF) for the oldest then LF
    ones.  (N == LF gives ones as well: the ramp is empty.)"""
    assert N >= 0
    if N == 0:
        return np.asarray([])
    if N < LF:
        return np.ones(N)
    ramp = np.linspace(1.0 / N, 1.0, num=N - LF)
    flat = np.ones(LF)
    return np.concatenate([ramp, flat], axis=0)


def n_below(n: int, gamma: float) -> int:
    return min(int(np.ceil(gamma * np.sqrt(n))), LF)


def ap_split_trials(losses, gamma: float):
    """hyperopt.tpe.ap_split_trials: the n_below = min(ceil(gamma·√n), 25) best trials (stable loss order, NumPy's order for
    non-finite losses: NaN last) are "below", the rest "above"; both index lists in told order."""
    losses = np.asarray(losses, dtype=np.float64)
    nb = n_below(len(losses), gamma)
    order = np.argsort(losses, kind="mergesort")
    keep = np.zeros(len(losses), dtype=bool)
    keep[order[:nb]] = True
    return np.flatnonzero(keep), np.flatnonzero(~keep)


def adaptive_parzen_normal(mus, prior_weight: float, prior_mu: float, prior_sigma: float, LF: int = LF):
    """hyperopt.tpe.adaptive_parzen_normal.  mus in told order.  Returns (weights, mus, sigmas) of the mixture: the sorted
    observations with the prior inserted at searchsorted(prior_mu) (n = 1: before the observation iff prior_mu < it),
    sigma = the larger gap to a neighbour (end points: their one gap; n = 1: prior_sigma / 2), clipped to
    [prior_sigma / min(100, 1 + #components), prior_sigma], the prior's sigma = prior_sigma; weights: linear forgetting by told
    order when n > LF (else ones), prior_weight for the prior, normalised."""
    mus = np.asarray(mus, dtype=np.float64)
    order = None
    if len(mus) == 0:
        srtd_mus = np.asarray([prior_mu], dtype=np.float64)
        sigma = np.asarray([prior_sigma], dtype=np.float64)
        prior_pos = 0
    elif len(mus) == 1:
        if prior_mu < mus[0]:
            prior_pos = 0
            srtd_mus = np.asarray([prior_mu, mus[0]])
            sigma = np.asarray([prior_sigma, prior_sigma * 0.5])
        else:
            prior_pos = 1
            srtd_mus = np.asarray([mus[0], prior_mu])
            sigma = np.asarray([prior_sigma * 0.5, prior_sigma])
        order = np.asarray([0])
    else:
        order = np.argsort(mus, kind="mergesort")
        prior_pos = int(np.searchsorted(mus[order], prior_mu))
        srtd_mus = np.zeros(len(mus) + 1)
        srtd_mus[:prior_pos] = mus[order[:prior_pos]]
        srtd_mus[prior_pos] = prior_mu
        srtd_mus[prior_pos + 1:] = mus[order[prior_pos:]]
        sigma = np.zeros_like(srtd_mus)
        sigma[1:-1] = np.maximum(srtd_mus[1:-1] - srtd_mus[0:-2], srtd_mus[2:] - srtd_mus[1:-1])
        sigma[0] = srtd_mus[1] - srtd_mus[0]
        sigma[-1] = srtd_mus[-1] - srtd_mus[-2]
    if LF and LF < len(mus):
        unsrtd_weights = linear_forgetting_weights(len(mus), LF)
        srtd_weights = np.zeros_like(srtd_mus)
        srtd_weights[:prior_pos] = unsrtd_weights[order[:prior_pos]]
        srtd_weights[prior_pos] = prior_weight
        srtd_weights[prior_pos + 1:] = unsrtd_weights[order[prior_pos:]]
    else:
        srtd_weights = np.ones(len(srtd_mus))
        srtd_weights[prior_pos] = prior_weight
    srtd_weights = srtd_weights / srtd_weights.sum()
    maxsigma = prior_sigma / 1.0
    minsigma = prior_sigma / min(100.0, (1.0 + len(srtd_mus)))
    sigma = np.clip(sigma, minsigma, maxsigma)
    sigma[prior_pos] = prior_sigma
    return srtd_weights, srtd_mus, sigma


def normal_cdf(x, mu, sigma):
    """hyperopt.tpe.normal_cdf."""
    top = np.asarray(x) - mu
    bottom = np.maximum(np.sqrt(2) * sigma, EPS)
    return 0.5 * (1 + erf(top / bottom))


def p_accept(weights, mus, sigmas, low, high):
    return np.sum(weights * (normal_cdf(high, mus, sigmas) - normal_cdf(low, mus, sigmas)))


def GMM1_lpdf(samples, weights, mus, sigmas, low, high, q=None):
    """hyperopt.tpe.GMM1_lpdf with both bounds.  Continuous: logsumexp over components of
    log(w / sqrt(2π σ²) / p_accept) - ½((x - μ) / max(σ, EPS))².  Quantized: log Σ w (Φ(min(x + q/2, hi)) - Φ(max(x - q/2, lo)))
    - log p_accept."""
    samples = np.asarray(samples, dtype=np.float64)
    weights, mus, sigmas = (np.asarray(a, dtype=np.float64) for a in (weights, mus, sigmas))
    pa = p_accept(weights, mus, sigmas, low, high)
    if q is None:
        dist = samples[:, None] - mus
        mahal = (dist / np.maximum(sigmas, EPS)) ** 2
        Z = np.sqrt(2 * np.pi * sigmas ** 2)
        coef = weights / Z / pa
        return logsum_rows(-0.5 * mahal + np.log(coef))
    prob = np.zeros(samples.shape, dtype=np.float64)
    for w, mu, sigma in zip(weights, mus, sigmas):
        ubound = np.minimum(samples + q / 2.0, high)
        lbound = np.maximum(samples - q / 2.0, low)
        inc_amt = w * normal_cdf(ubound, mu, sigma)
        inc_amt -= w * normal_cdf(lbound, mu, sigma)
        prob += inc_amt
    return np.log(prob) - np.log(pa)


def logsum_rows(x):
    """hyperopt.tpe.logsum_rows."""
    m = x.max(axis=1)
    return np.log(np.exp(x - m[:, None]).sum(axis=1)) + m


def GMM1_raw(weights, mus, sigmas, low, high, rng, size):
    """hyperopt.tpe.GMM1's bounded draw, before quantization: pick a component ∝ w, draw from it, keep the draw iff
    low <= x < high (rejection; vectorised in rounds, same distribution as hyperopt's one-at-a-time loop)."""
    out = np.empty(0)
    w = np.asarray(weights, dtype=np.float64)
    while out.size < size:
        n = max(2 * (size - out.size), 64)
        k = rng.choice(len(w), size=n, p=w / w.sum())
        x = rng.normal(loc=np.asarray(mus)[k], scale=np.asarray(sigmas)[k])
        out = np.concatenate([out, x[(low <= x) & (x < high)]])
    return out[:size]


def quantize(x, q):
    """hyperopt's rounding of quantized draws: np.round(x / q) * q (round half to even)."""
    return np.round(np.asarray(x) / q) * q


def truncated_mixture_cdf(x, weights, mus, sigmas, low, high):
    """CDF of the mixture truncated to [low, high) — the distribution GMM1_raw samples."""
    x = np.asarray(x, dtype=np.float64)
    num = (weights * (normal_cdf(x[..., None], mus, sigmas) - normal_cdf(low, mus, sigmas))).sum(-1)
    return num / p_accept(weights, mus, sigmas, low, high)


def ap_categorical_tables(obs, prior_weight: float, upper: int, LF: int = LF):
    """hyperopt.tpe.ap_categorical_sampler's probabilities: bincount(obs, linear-forgetting weights) + prior_weight,
    normalised [RECALL: the pseudocount is prior_weight per category]."""
    obs = np.asarray(obs, dtype=np.int64)
    weights = linear_forgetting_weights(len(obs), LF=LF)
    counts = np.bincount(obs, minlength=upper, weights=weights) if len(obs) else np.zeros(upper)
    pseudocounts = counts + prior_weight
    return pseudocounts / pseudocounts.sum()


def build_models(space, X, losses, gamma: float = 0.25, prior_weight: float = 1.0):
    """The below / above models of every parameter (hyperopt.tpe.build_posterior for a flat space).  X: n × D in parameter
    units (category indices for choices), told order.  Returns (list of per-parameter dicts, n_below)."""
    X = np.asarray(X, dtype=np.float64).reshape(-1, len(space))
    below, above = ap_split_trials(losses, gamma)
    models = []
    for d, p in enumerate(space):
        if p[0] == "choice":
            models.append(dict(kind="choice", below=ap_categorical_tables(X[below, d], prior_weight, p[1]),
                               above=ap_categorical_tables(X[above, d], prior_weight, p[1])))
            continue
        lo, hi = float(p[1]), float(p[2])
        pm, ps = 0.5 * (hi + lo), 1.0 * (hi - lo)
        m = dict(kind=p[0], lo=lo, hi=hi, q=float(p[3]) if p[0] == "quniform" else None)
        for name, idx in (("below", below), ("above", above)):
            w, mu, sg = adaptive_parzen_normal(X[idx, d], prior_weight, pm, ps)
            m[name] = dict(w=w, mu=mu, sigma=sg, p_accept=p_accept(w, mu, sg, lo, hi))
        models.append(m)
    return models, len(below)


def score(model, cand):
    """log l(x) - log g(x) of every candidate (numeric: values before quantization; choices: category indices)."""
    cand = np.asarray(cand, dtype=np.float64)
    if model["kind"] == "choice":
        c = cand.astype(np.int64)
        return np.log(model["below"][c]) - np.log(model["above"][c])
    x = quantize(cand, model["q"]) if model["q"] is not None else cand
    b, a = model["below"], model["above"]
    return (GMM1_lpdf(x, b["w"], b["mu"], b["sigma"], model["lo"], model["hi"], model["q"])
            - GMM1_lpdf(x, a["w"], a["mu"], a["sigma"], model["lo"], model["hi"], model["q"]))


def draw(model, M: int, rng):
    """M candidates from the below model (numeric: before quantization; choices: category indices), hyperopt's way."""
    if model["kind"] == "choice":
        return rng.choice(len(model["below"]), size=M, p=model["below"]).astype(np.float64)
    b = model["below"]
    return GMM1_raw(b["w"], b["mu"], b["sigma"], model["lo"], model["hi"], rng, M)


def choose(models, cands):
    """hyperopt's per-parameter decision: for each parameter the candidate at np.argmax of its scores (first index of the
    maximum).  cands: D arrays of candidates.  Returns (values, indices); quantized values are rint(x/q)·q."""
    vals, idxs = [], []
    for m, c in zip(models, cands):
        i = int(np.argmax(score(m, c)))
        v = float(c[i])
        if m["kind"] == "quniform":
            v = float(quantize(v, m["q"]))
        vals.append(v)
        idxs.append(i)
    return np.asarray(vals), np.asarray(idxs)
