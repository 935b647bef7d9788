"""An FP64 torch restatement of oracle/mvtpe_oracle.score for the exhaustive checks of tests/test_gpu_mvtpe.py: every candidate
of a 2^20 set against 8 193 components is too much for NumPy in a test, not for the device.  Uses nothing from libkbo.  Pinned
to the NumPy oracle by tests/test_mvtpe_oracle.py (on the CPU device)."""
import math

import numpy as np
import torch

from oracle import mvtpe_oracle as O

R2 = 1.0 / math.sqrt(2.0)


def log_gauss_mass(a, b):
    """oracle.mvtpe_oracle.log_gauss_mass in torch, elementwise, a < b."""
    right = a > 0
    a, b = torch.where(right, -b, a), torch.where(right, -a, b)
    left = b <= 0
    la, lb = torch.special.log_ndtr(a), torch.special.log_ndtr(b)
    tail = lb + torch.log(-torch.expm1(torch.clamp(la - lb, max=-1e-300)))
    central = torch.log(0.5 * (torch.erf(b * R2) + torch.erf(-a * R2)))
    return torch.where(left, tail, central)


def _group_terms(space, g, device):
    """Per component (observations, then the prior) the constants that do not depend on the candidate."""
    m = len(g["w"]) - 1
    out = []
    for d, p in enumerate(space):
        if p[0] == "cat":
            out.append(None)
            continue
        lo, hi, lo2, hi2, q = O.bounds(p)
        mus = np.append(g["mu"][:, d], 0.5 * (lo2 + hi2))
        sgs = np.append(np.full(m, g["sigma"][d]), hi2 - lo2)
        lz = O.log_gauss_mass((lo2 - mus) / sgs, (hi2 - mus) / sgs)
        out.append(tuple(torch.tensor(v, dtype=torch.float64, device=device) for v in (mus, sgs, lz)))
    return out


def log_density(space, g, cands, chunk=2048):
    """oracle.mvtpe_oracle.log_density: cands is an (M × D) float64 tensor; returns (M,) float64."""
    dev = cands.device
    terms = _group_terms(space, g, dev)
    m = len(g["w"]) - 1
    lw = torch.tensor(np.log(g["w"]), dtype=torch.float64, device=dev)
    obs = torch.tensor(g["mu"], dtype=torch.float64, device=dev)
    res = []
    for s in range(0, cands.shape[0], chunk):
        x = cands[s:s + chunk]
        t = lw.expand(x.shape[0], m + 1).clone()
        for d, p in enumerate(space):
            xd = x[:, d:d + 1]
            if p[0] == "cat":
                C = p[1]
                hit = xd == obs[:, d][None, :]
                lr = math.log(g["cat_rows"][d, 1])
                t[:, :m] += lr + hit.to(torch.float64) * (math.log(g["cat_rows"][d, 0]) - lr)
                t[:, m] -= math.log(C)
                continue
            mus, sgs, lz = terms[d]
            if p[0] == "float":
                z = (xd - mus) / sgs
                t += -0.5 * z * z - O.LN_SQRT_2PI - torch.log(sgs) - lz
            else:
                lo, hi, lo2, hi2, q = O.bounds(p)
                xl, xu = torch.clamp(xd - 0.5 * q, min=lo2), torch.clamp(xd + 0.5 * q, max=hi2)
                t += log_gauss_mass((xl - mus) / sgs, (xu - mus) / sgs) - lz
        res.append(torch.logsumexp(t, dim=1))
    return torch.cat(res)


def score(space, models, cands, chunk=2048):
    return log_density(space, models["below"], cands, chunk) - log_density(space, models["above"], cands, chunk)
