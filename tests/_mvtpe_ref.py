"""An FP64 torch restatement of oracle/mvtpe_oracle.score for the exhaustive checks of tests/test_gpu_mvtpe.py and
tests/test_gpu_mvtpe_scale.py: every candidate of a 2^20 set against 8 193 components is too much for NumPy in a test, not for
the device.  Uses nothing from libkbo.  Pinned to the NumPy oracle by tests/test_mvtpe_oracle.py (on the CPU device).

Besides the scores, ``tol`` gives per candidate how far two correct FP64 evaluations of the same score can lie apart (this one
and the engine's, with its models equal to the oracle's to a few ulps), so that a decision check can tell a wrong pick from a
near-tie that rounding may break either way; ``pick_ok`` is that check."""
import math

import numpy as np
import torch

from oracle import mvtpe_oracle as O

R2 = 1.0 / math.sqrt(2.0)
U = 2.0 ** -53                    # unit roundoff of FP64


def log_gauss_mass(a, b):
    """oracle.mvtpe_oracle.log_gauss_mass in torch, elementwise, a < b."""
    right = a > 0
    a, b = torch.where(right, -b, a), torch.where(right, -a, b)
    left = b <= 0
    la, lb = torch.special.log_ndtr(a), torch.special.log_ndtr(b)
    tail = lb + torch.log(-torch.expm1(torch.clamp(la - lb, max=-1e-300)))
    central = torch.log(0.5 * (torch.erf(b * R2) + torch.erf(-a * R2)))
    return torch.where(left, tail, central)


def _group_terms(space, g):
    """Per component (observations, then the prior) the part of its log density that does not depend on the candidate, c_k:
    log w_k, per float −log(σ√2π) − log of its truncation mass, per integer −log of its truncation mass, per categorical the
    row's entry off the observed category (1/C for the prior); and |c|_k, the same terms' magnitudes summed.  Then per
    parameter what the candidate meets: (means, sigmas) of a float or an integer, a categorical's match bonus."""
    m = len(g["w"]) - 1
    lw = np.log(g["w"])
    c, mag = lw.copy(), np.abs(lw)
    par = []
    for d, p in enumerate(space):
        if p[0] == "cat":
            lm, lr = math.log(g["cat_rows"][d, 0]), math.log(g["cat_rows"][d, 1])
            c[:m] += lr
            c[m] -= math.log(p[1])
            mag[:m] += abs(lr)
            mag[m] += math.log(p[1])
            par.append(lm - lr)
            continue
        lo, hi, lo2, hi2, q = O.bounds(p)
        mus = np.append(g["mu"][:, d], 0.5 * (lo2 + hi2))
        sgs = np.append(np.full(m, g["sigma"][d]), hi2 - lo2)
        lz = O.log_gauss_mass((lo2 - mus) / sgs, (hi2 - mus) / sgs)
        if p[0] == "float":
            c += -O.LN_SQRT_2PI - np.log(sgs) - lz
            mag += O.LN_SQRT_2PI + np.abs(np.log(sgs)) + np.abs(lz)
        else:
            c -= lz
            mag += np.abs(lz)
        par.append((mus, sgs))
    return c, mag, par


def log_density(space, g, cands, chunk=2048):
    """oracle.mvtpe_oracle.log_density: cands is an (M × D) float64 tensor; returns (M,) float64.  Each component's
    exponent is c_k plus, per parameter, −½z² (float), the log mass of the candidate's bin (integer) or the match bonus
    (categorical)."""
    dev = cands.device
    c, _, par = _group_terms(space, g)
    m = len(g["w"]) - 1
    c = torch.tensor(c, dtype=torch.float64, device=dev)
    par = [v if isinstance(v, float) else tuple(torch.tensor(a, dtype=torch.float64, device=dev) for a in v) for v in par]
    obs = torch.tensor(g["mu"], dtype=torch.float64, device=dev)
    res = []
    for s in range(0, cands.shape[0], chunk):
        x = cands[s:s + chunk]
        t = c.expand(x.shape[0], m + 1).clone()
        for d, p in enumerate(space):
            xd = x[:, d:d + 1]
            if p[0] == "cat":
                t[:, :m].add_((xd == obs[:, d][None, :]).to(torch.float64), alpha=par[d])
                continue
            mus, sgs = par[d]
            if p[0] == "float":
                z = (xd - mus).div_(sgs)
                t.addcmul_(z, z, value=-0.5)
            else:
                lo, hi, lo2, hi2, q = O.bounds(p)
                xl, xu = torch.clamp(xd - 0.5 * q, min=lo2), torch.clamp(xd + 0.5 * q, max=hi2)
                t += log_gauss_mass((xl - mus) / sgs, (xu - mus) / sgs)
        res.append(torch.logsumexp(t, dim=1))
    return torch.cat(res)


def score(space, models, cands, chunk=2048):
    return log_density(space, models["below"], cands, chunk) - log_density(space, models["above"], cands, chunk)


# ---- how far two FP64 evaluations of a score can differ ------------------------------------------------------------------
# One group, L = log Σ_k exp(t_k), t_k = c_k + v_k, v_k = −Σ_float ½z² + Σ_int (log bin mass) + Σ_cat b·[match].  Either
# evaluation sums about 4D + 2 terms into t_k (the engine: c_k's 3 per parameter, then one per parameter at the candidate; this
# file: c_k's, then one per parameter), each term carrying a few roundings of its own and the models' few-ulp differences
# (σ, the weights), so t_k is off by at most (4D + 16)u·(|c|_k + |v_k|).  Log-sum-exp moves by the softmax-weighted
# average p_k of those, and Σ_k p_k|v_k| ≤ V = C_max + 2B + log(m + 1) − L (B = Σ match bonuses): the v_k are ≤ 0 but for
# the bonuses, and Σ_k p_k t_k = L − H(p) ≥ L − log(m + 1).  An integer bin far in a tail is a difference of two log Φ, whose
# few-ulp errors are amplified by σ/q: ≤ 4u(1 + |log mass|)(1 + σ/q) per term, ≤ 4u(1 + σ/q)(n_int + V) in all.  The sums
# of m + 1 exponentials and the final log: (m + 4)u + 2u|L|.  Two evaluations, and the engine's weights normalised by a
# sum in another order ((m + 2)u):
#   T_g = 2[(4D + 16)u(max_k |c|_k + V) + 4u(1 + σ/q)(n_int + V) + (m + 4)u + 2u|L|] + (m + 2)u.
# A score's tolerance is the sum over its two groups.
def _group_tol(space, g, L):
    c, mag, par = _group_terms(space, g)
    m, D = len(g["w"]) - 1, len(space)
    B = sum(v for v in par if isinstance(v, float))
    ints = [d for d, p in enumerate(space) if p[0] == "int"]
    amp = max((g["sigma"][d] / O.bounds(space[d])[4] for d in ints), default=0.0)
    V = (float(c.max()) + 2 * B + math.log(m + 1) - L).clamp_(min=0.0)
    e1 = (4 * D + 16) * U * (float(mag.max()) + V) + (4 * U * (1 + amp) * (len(ints) + V) if ints else 0.0) \
        + (m + 4) * U + 2 * U * L.abs()
    return 2 * e1 + (m + 2) * U


def score_tol(space, models, cands, chunk=2048):
    """(score, tol) of every candidate, each group's log density evaluated once."""
    Lb, La = (log_density(space, models[g], cands, chunk) for g in ("below", "above"))
    return Lb - La, _group_tol(space, models["below"], Lb) + _group_tol(space, models["above"], La)


def tol(space, models, cands, chunk=2048):
    return score_tol(space, models, cands, chunk)[1]


def pick_ok(cands, s, T, idx):
    """Whether the engine's pick idx among the candidates (M × D, as scored), scored s with tolerances T by this reference,
    is np.argmax's: the first occurrence of the best candidate, wherever no other candidate lies within the two evaluations'
    tolerances of the maximum; else a candidate within them, at its first occurrence.  Returns (ok, message, number of
    distinct candidates in that tie band)."""
    best = int(torch.argmax(s))                                      # the first index of the maximum
    smax = s[best]
    band = torch.nonzero(s >= smax - T - T[best]).flatten()
    first = lambda i: int(torch.nonzero((cands == cands[i]).all(dim=1)).flatten()[0])
    keys = len(torch.unique(cands[band], dim=0))
    if keys == 1:
        want = first(best)
        return idx == want, f"pick {idx}, reference first maximum {want} (score {float(smax):.17g})", 1
    ok = bool((band == idx).any()) and first(idx) == idx
    return ok, (f"pick {idx} (score {float(s[idx]):.17g}) is not the first occurrence of a candidate within tolerance of the "
                f"reference maximum {float(smax):.17g} at {best}"), keys
