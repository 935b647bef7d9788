"""The GP posterior over a whole candidate grid in FP64, with torch alone: the reference test_gpu_grid_scale.py holds the engine to.

Nothing here touches libkbo.  Formula for formula it is oracle/gp_oracle.py (gp_fit, gp_predict, acquisition), run through torch
so that it can take a million candidates at N = 8192 on the GPU (device="cuda") and pin itself against the oracle on the CPU
(device="cpu", tests/test_posterior_ref.py):
  * y normalised by its mean and population std, with scikit-learn's zero-std guard (std < 10·eps -> 1);
  * X and Xc divided by ℓ (a scalar or one value per dimension), squared distances formed by exact differences summed over the
    dimensions (scipy cdist's arithmetic) — never as ‖a‖² + ‖b‖² − 2a·b, which cancels next to a trial point;
  * L = cholesky(amplitude·k(X, X) + noise·I), α = cholesky_solve(L, yn);
  * per chunk of candidates: μ = K*·α, V = solve_triangular(L, K*ᵀ), σ² = amplitude − Σ V² clamped at 0, both un-normalised
    (predict_normalised: μ_n, σ²_n unclamped and the prefix variances amplitude − Σ_{j<P} V_j², in normalised units);
  * EI / LCB / PI by oracle.acquisition on the host with y_opt = min(y).
Float32 candidates are widened to float64 before anything else, as the engine widens them.  Temporaries stay under
``budget`` bytes (2 GiB by default), whatever the grid.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import gp_oracle as O

ACQS = ("ei", "lcb", "pi")


def _f64(A, device):
    """A NumPy array or a tensor (float32 or float64, any device) as a float64 tensor on `device`."""
    if isinstance(A, torch.Tensor):
        return A.to(device=device, dtype=torch.float64)
    return torch.as_tensor(np.asarray(A)).to(device=device, dtype=torch.float64)


def kernel(As, Bs, kind, amplitude, budget):
    """amplitude·k(As, Bs) of length-scaled rows: squared distances by exact differences, (rows, |Bs|, D) at a time."""
    n, D = Bs.shape
    out = torch.empty(As.shape[0], n, dtype=torch.float64, device=As.device)
    step = max(1, budget // (8 * n * D))
    for r0 in range(0, As.shape[0], step):
        d2 = (As[r0:r0 + step, None, :] - Bs[None, :, :]).square_().sum(-1)
        if kind == O.KERNEL_RBF:
            k = torch.exp(-0.5 * d2)
        elif kind == O.KERNEL_MATERN52:
            s = torch.sqrt(d2) * math.sqrt(5.0)
            k = (1.0 + s + s * s / 3.0) * torch.exp(-s)
        else:
            raise ValueError(f"unknown kernel {kind!r}")
        out[r0:r0 + step] = amplitude * k
    return out


def fit(X, y, *, kind, length_scale, amplitude, noise, normalize_y=True, device="cuda", budget=2 << 30):
    """oracle.gp_fit in torch: the normalised targets, L, α and the LML."""
    y = _f64(y, device).reshape(-1)
    if normalize_y:
        y_mean = float(y.mean())
        y_std = float(y.std(correction=0))
        if y_std < 10 * np.finfo(np.float64).eps:
            y_std = 1.0
    else:
        y_mean, y_std = 0.0, 1.0
    ls = _f64(np.atleast_1d(np.asarray(length_scale, dtype=np.float64)), device)
    Xs = _f64(X, device) / ls
    yn = (y - y_mean) / y_std
    K = kernel(Xs, Xs, kind, amplitude, budget // 2)
    K.diagonal().add_(noise)
    L = torch.linalg.cholesky(K)
    del K
    alpha = torch.cholesky_solve(yn[:, None], L)[:, 0]
    lml = float(-0.5 * (yn @ alpha) - torch.log(torch.diagonal(L)).sum() - 0.5 * len(yn) * np.log(2 * np.pi))
    return dict(Xs=Xs, ls=ls, L=L, alpha=alpha, y_mean=y_mean, y_std=y_std, y_opt=float(y.min()), kind=kind,
                amplitude=float(amplitude), lml=lml, budget=budget)


def _chunks(f, Xc, prefixes=()):
    """Per chunk of rows of Xc: (first row, μ_n = K*·α, σ²_n = amplitude − Σ V² unclamped, {P: amplitude − Σ_{j<P} V_j²}), all in
    normalised units, as float64 tensors on the fit's device; chunks sized so that K*, V and the distance temporaries fit the
    fit's budget."""
    dev = f["L"].device
    N, D = f["Xs"].shape
    M = Xc.shape[0]
    rows = max(1, f["budget"] // (4 * 8 * N))          # K*, V, and a quarter for the distance slabs and the row sums
    for c0 in range(0, M, rows):
        A = _f64(Xc[c0:c0 + rows], dev) / f["ls"]
        Ks = kernel(A, f["Xs"], f["kind"], f["amplitude"], f["budget"] // 4)
        m = Ks @ f["alpha"]
        V = torch.linalg.solve_triangular(f["L"], Ks.T, upper=False)
        del Ks
        V.square_()
        var_p = {P: f["amplitude"] - V[:P].sum(0) for P in prefixes}
        var = f["amplitude"] - V.sum(0)
        del V
        yield c0, m, var, var_p


def predict(f, Xc):
    """oracle.gp_predict in torch: μ and σ of every row of Xc (host float64 arrays)."""
    M = Xc.shape[0]
    mu = np.empty(M)
    std = np.empty(M)
    for c0, m, var, _ in _chunks(f, Xc):
        var.clamp_(min=0.0)
        mu[c0:c0 + len(m)] = (f["y_std"] * m + f["y_mean"]).cpu().numpy()
        std[c0:c0 + len(m)] = torch.sqrt(var * f["y_std"] ** 2).cpu().numpy()
    return mu, std


def predict_normalised(f, Xc, prefixes=()):
    """What the sweep's ranking arithmetic approximates, in normalised units (host float64 arrays): dict(mu_n = K*·α, var_n =
    amplitude − Σ V² before any clamp, var_p = {P: amplitude − Σ_{j<P} V_j²}).  V = L⁻¹K*ᵀ, and its first P rows depend on
    L[:P, :P] alone, so var_p[P] is the exact posterior variance given the first P trials: the upper bound a sweep forms from a
    prefix of the trials.  It does not increase with P, and var_p[N] is var_n."""
    M = Xc.shape[0]
    out = dict(mu_n=np.empty(M), var_n=np.empty(M), var_p={P: np.empty(M) for P in prefixes})
    for c0, m, var, var_p in _chunks(f, Xc, prefixes):
        r = slice(c0, c0 + len(m))
        out["mu_n"][r] = m.cpu().numpy()
        out["var_n"][r] = var.cpu().numpy()
        for P, v in var_p.items():
            out["var_p"][P][r] = v.cpu().numpy()
    return out


def top2(a):
    """(first argmax, its value, the best value at any other row)."""
    i = int(np.argmax(a))
    v = float(a[i])
    rest = a.copy()
    rest[i] = -np.inf
    return i, v, float(np.max(rest))


def acquisitions(mu, std, y_opt, *, xi, kappa):
    """EI, LCB and PI of the whole grid (oracle.acquisition, values to maximise) and each one's top-1 / top-2."""
    out = {a: O.acquisition(mu, std, y_opt, a, xi, kappa) for a in ACQS}
    return out, {a: top2(out[a]) for a in ACQS}


def posterior(X, y, Xc, *, kind, length_scale, amplitude, noise, xi, kappa, normalize_y=True, device="cuda", budget=2 << 30):
    """fit + predict + acquisitions: dict(mu, std, acq={ei, lcb, pi}, top={acq: (index, value, next best)}, fit)."""
    f = fit(X, y, kind=kind, length_scale=length_scale, amplitude=amplitude, noise=noise, normalize_y=normalize_y, device=device,
            budget=budget)
    mu, std = predict(f, Xc)
    acq, top = acquisitions(mu, std, f["y_opt"], xi=xi, kappa=kappa)
    return dict(mu=mu, std=std, acq=acq, top=top, fit=f)
