"""An FP64 torch restatement of oracle/tpe_oracle.score for the exhaustive checks of tests/test_gpu_tpe_scale.py and
tests/test_gpu_tpe.py: every candidate of a 2^20 set against 8 193 components is too much for NumPy in a test, not for the
device.  The models come from oracle.tpe_oracle.build_models (NumPy); nothing here uses libkbo.  Pinned to the NumPy oracle by
tests/test_tpe_ref.py (on the CPU device).

Besides the scores, ``tol`` gives per candidate how far two correct FP64 evaluations of the same score can lie apart (this one
and the engine's, with its models equal to the oracle's to a few ulps), so that a decision check can tell a wrong pick from a
near-tie that rounding may break either way; ``pick_ok`` is that check."""
import math

import numpy as np
import torch

from oracle import tpe_oracle as O

U = 2.0 ** -53                    # unit roundoff of FP64
BUDGET = 1 << 27                  # candidates × components per chunk: 1 GiB per FP64 temporary, a few of them live at once


def _t(a, dev):
    return torch.as_tensor(np.asarray(a, dtype=np.float64), device=dev)


def _rows(nc):
    return max(1, BUDGET // max(nc, 1))


def _cont_consts(g, dev):
    """(mu, max(sigma, EPS), log coef) of one continuous group, the coefficient formed as GMM1_lpdf forms it."""
    w, mu, sg = (np.asarray(g[k], dtype=np.float64) for k in ("w", "mu", "sigma"))
    lc = np.log(w / np.sqrt(2 * np.pi * sg ** 2) / g["p_accept"])
    return _t(mu, dev), _t(np.maximum(sg, O.EPS), dev), _t(lc, dev)


def cont_lpdf(g, x):
    """GMM1_lpdf of one continuous group (dict w, mu, sigma, p_accept) at the candidates x ((M,) float64 tensor):
    logsumexp_k(log(w_k / sqrt(2π σ_k²) / p_accept) − ½((x − μ_k) / max(σ_k, 1e-12))²)."""
    mu, sd, lc = _cont_consts(g, x.device)
    out = torch.empty_like(x)
    c = _rows(len(mu))
    for s in range(0, x.shape[0], c):
        z = (x[s:s + c, None] - mu).div_(sd)
        out[s:s + c] = torch.logsumexp(torch.addcmul(lc, z, z, value=-0.5), dim=1)
    return out


def _phi(x, mu, den):
    """hyperopt's normal_cdf with den = max(√2·σ, EPS)."""
    return 0.5 * (1.0 + torch.erf((x - mu) / den))


def quant_terms(g, v, lo, hi, q):
    """Of one quantized group at the quantized values v: (GMM1_lpdf, Σ_k w_k (Φ_k(ub) − Φ_k(lb))), ub = min(v + q/2, hi),
    lb = max(v − q/2, lo)."""
    dev = v.device
    w, mu = _t(g["w"], dev), _t(g["mu"], dev)
    den = _t(np.maximum(np.sqrt(2) * np.asarray(g["sigma"], dtype=np.float64), O.EPS), dev)
    lpdf, prob = torch.empty_like(v), torch.empty_like(v)
    c = _rows(len(w))
    for s in range(0, v.shape[0], c):
        ub = torch.clamp(v[s:s + c] + q / 2.0, max=hi)[:, None]
        lb = torch.clamp(v[s:s + c] - q / 2.0, min=lo)[:, None]
        p = (w * _phi(ub, mu, den) - w * _phi(lb, mu, den)).sum(dim=1)
        prob[s:s + c] = p
        lpdf[s:s + c] = torch.log(p) - math.log(g["p_accept"])
    return lpdf, prob


def quantize(model, x):
    return torch.round(x / model["q"]) * model["q"]           # np.round and torch.round both round half to even


def score(model, x):
    """oracle.tpe_oracle.score: log l(x) − log g(x) of every candidate ((M,) float64 tensor; numeric values before
    quantization, category indices for choices)."""
    if model["kind"] == "choice":
        c = x.to(torch.int64)
        return torch.log(_t(model["below"], x.device)[c]) - torch.log(_t(model["above"], x.device)[c])
    b, a = model["below"], model["above"]
    if model["q"] is None:
        return cont_lpdf(b, x) - cont_lpdf(a, x)
    v = quantize(model, x)
    return quant_terms(b, v, model["lo"], model["hi"], model["q"])[0] - quant_terms(a, v, model["lo"], model["hi"], model["q"])[0]


def key(model, x):
    """What the score depends on: the level of a quantized candidate, else the candidate itself."""
    return quantize(model, x) if model["kind"] == "quniform" else x


# ---- how far two FP64 evaluations of a score can differ ------------------------------------------------------------------
# Continuous, one group, L = log Σ_k exp(t_k), t_k = lc_k − ½z_k²: each evaluation forms z_k = (x − μ_k)/σ_k with 2 roundings,
# z_k² and the fma or add with lc_k with 2 more and lc_k itself (log of w/√(2πσ²)/p_accept) with about 4, so t_k is off by at
# most 6u(|lc_k| + ½z_k²); log-sum-exp moves by the p_k = softmax(t)_k-weighted average of those.  Each sum of nc exponentials
# carries at most nc + 2 roundings (exp's own error included), and the engine's weights, normalised by a sum taken in another
# order, move lc_k by at most nc·u.  The final log and add: 2u|L| each.  Two evaluations:
#   T_g = 12u·Σ_k p_k(|lc_k| + ½z_k²) + (3nc + 4)u + 4u|L|,  rounded up to 16u in the first term.
# Quantized, one group: each Φ_k is formed from erf with an absolute error of a few ulps of 1 (≤ 4u after the halving, the
# add of 1 and the product with w_k), so each evaluation's Σ_k w_k(Φ_k(ub) − Φ_k(lb)) is off by ≤ 8u·Σw absolutely and by
# (nc + 2)u relatively from the summation; the log turns that into 16u·Σw / Σw(Φ(ub) − Φ(lb)) + (3nc + 4)u for two of them.
# A score's tolerance is the sum over its two groups.  Choice scores are a table lookup: 0.
def _cont_tol(g, x):
    mu, sd, lc = _cont_consts(g, x.device)
    nc = len(mu)
    out = torch.empty_like(x)
    c = _rows(nc)
    for s in range(0, x.shape[0], c):
        z = (x[s:s + c, None] - mu).div_(sd)
        t = torch.addcmul(lc, z, z, value=-0.5)
        L = torch.logsumexp(t, dim=1)
        p = torch.softmax(t, dim=1)
        spread = (p * (lc.abs() - t + lc)).sum(dim=1)             # Σ p_k (|lc_k| + ½z_k²)
        out[s:s + c] = 16 * U * spread + (3 * nc + 4) * U + 4 * U * L.abs()
    return out


def _cont_tol_cap(g, x):
    """An upper bound on _cont_tol over every candidate in [x.min(), x.max()]: ½z² ≤ ½zmax², |L| ≤ max|lc| + ½zmax² + log nc."""
    mu, sd, lc = _cont_consts(g, x.device)
    zmax = float(torch.maximum((x.max() - mu).abs(), (x.min() - mu).abs()).div(sd).max())
    a = float(lc.abs().max()) + 0.5 * zmax * zmax
    return 16 * U * a + (3 * len(mu) + 4) * U + 4 * U * (a + math.log(len(mu)))


def tol(model, x):
    if model["kind"] == "choice":
        return torch.zeros_like(x)
    b, a = model["below"], model["above"]
    if model["q"] is None:
        return _cont_tol(b, x) + _cont_tol(a, x)
    v = quantize(model, x)
    out = torch.zeros_like(x)
    for g in (b, a):
        _, prob = quant_terms(g, v, model["lo"], model["hi"], model["q"])
        out += 16 * U * float(np.sum(g["w"])) / prob + (3 * len(g["w"]) + 4) * U
    return out


def pick_ok(model, x, s, idx):
    """Whether the engine's pick idx among the candidates x (scored s by this reference) is np.argmax's: the first candidate
    with the best key, wherever no candidate of another key lies within the two evaluations' tolerances of the maximum; else
    a candidate within them, at the first occurrence of its key.  Returns (ok, message, number of keys in that tie band)."""
    best = int(torch.argmax(s))                                      # the first index of the maximum
    smax = s[best]
    if model["kind"] == "choice":                                     # exact scores: np.argmax itself
        return idx == best, f"pick {idx}, reference first maximum {best} (score {float(smax):.17g})", 1
    if model["kind"] == "uniform":
        cap = _cont_tol_cap(model["below"], x) + _cont_tol_cap(model["above"], x)
        near = torch.nonzero(s >= smax - 2 * cap).flatten()
    else:
        near = torch.arange(x.shape[0], device=x.device)
    T = tol(model, x[near])
    Tb = float(T[near == best][0])
    band = near[s[near] >= smax - T - Tb]
    k = key(model, x)
    first = lambda i: int(torch.nonzero(k == k[i]).flatten()[0])
    keys = torch.unique(k[band])
    if len(keys) == 1:
        want = first(best)
        return idx == want, f"pick {idx}, reference first maximum {want} (score {float(smax):.17g})", 1
    ok = bool((band == idx).any()) and first(idx) == idx
    return ok, (f"pick {idx} (score {float(s[idx]):.17g}) is not the first occurrence of a candidate within tolerance of the "
                f"reference maximum {float(smax):.17g} at {best}"), len(keys)
