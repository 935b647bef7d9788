"""CPU oracle for CMA-ES with learning-rate adaptation (LRA-CMA-ES; M. Nomura, Y. Akimoto, I. Ono, "CMA-ES with Learning
Rate Adaptation: Can CMA-ES with Default Population Size Solve Multimodal and Noisy Problems?", GECCO 2023), as
CyberAgent's ``cmaes`` library implements it and Optuna's ``CmaEsSampler(lr_adapt=True)`` uses it: Katib ``cmaes`` with
``lr_adapt: true``.  Builds on ``cma_oracle.CmaState`` / ``tell`` and leaves them unchanged.

TEST INFRASTRUCTURE ONLY, FP64 NumPy.  PARITY UNPINNED: neither ``cmaes`` nor Optuna is available offline, so every rule
below is written from memory and marked [RECALL]; where memory and the paper disagree, the paper wins.

1. Constants [RECALL]: α = 1.4, β_m = 0.1, β_Σ = 0.03, γ = 0.1.  State: E_m ∈ ℝ^D, E_Σ ∈ ℝ^{D×D}, V_m, V_Σ, all 0, and
   η_m = η_Σ = 1 at the start of a run.
2. A tell [RECALL] first runs the plain update (``cma_oracle.tell``: paths, σ′, C′ from m, σ, C), then
   Δm = m′ − m and ΔΣ = σ′²C′ − σ²C; with P = Σ^{-1/2} = B diag(1/d) Bᵀ/σ from C's eigendecomposition before the tell,
   Δ̃m = P·Δm and Δ̃Σ = P·ΔΣ·P/√2.
3. Moving averages [RECALL]: E ← (1 − β)·E + β·Δ̃, V ← (1 − β)·V + β·‖Δ̃‖² (Frobenius for Σ), with β_m or β_Σ.
4. SNR = (‖E‖² − β/(2 − β)·V)/(V − ‖E‖²); η ← η·exp(min(γη, β)·clip(SNR/(αη) − 1, −1, 1)), then η ← min(η, 1).
5. m ← m + η_m·Δm, Σ ← σ²C + η_Σ·ΔΣ; σ ← exp(Σ_j log λ_j(Σ)/(2D)), capped at 1e32; C ← Σ/σ², so det C = 1; and last
   σ ← σ·η_m(before step 4)/η_m(after).
A restart starts a fresh LRA state, as a fresh ``CMA(lr_adapt=True)`` would.  The evolution paths and the termination test
are the plain ones.

Stated departures:
(a) When V − ‖E‖² is not positive and finite, that η stays unchanged (upstream divides by zero and the run turns NaN).
(b) The log-determinant is taken from the eigenvalues of Σ/σ′² (σ′ the plain update's step size, the matrix the device
    decomposes) plus 2D·log σ′, and an eigenvalue ≤ 0 is floored at ``cma_oracle.EPS`` as ``cma_oracle.eigen`` floors.
    With η_Σ ≤ 1, Σ is a convex combination of two SPD matrices, so only rounding can get there.
(c) ``lr_adapt`` beside ``with_margin`` is refused, as Optuna refuses it [RECALL]; beside ``restart_strategy`` it is
    allowed (Optuna's restarts are a different mechanism [RECALL], so it may refuse a combination this service allows).
"""
from __future__ import annotations

import numpy as np

from . import cma_oracle as O

ALPHA, BETA_MEAN, BETA_SIGMA, GAMMA = 1.4, 0.1, 0.03, 0.1
SIGMA_MAX = 1e32


class LraState:
    """E, V and η of one run (item 1)."""

    def __init__(self, D: int):
        self.E_mean = np.zeros(D)
        self.E_Sigma = np.zeros((D, D))
        self.V_mean = 0.0
        self.V_Sigma = 0.0
        self.eta_mean = 1.0
        self.eta_Sigma = 1.0


def snr(E2: float, V: float, beta: float):
    """Item 4's SNR from ‖E‖² and V, or None when V − ‖E‖² is not positive and finite (departure (a))."""
    den = V - E2
    if not (np.isfinite(den) and den > 0.0):
        return None
    return (E2 - beta / (2.0 - beta) * V) / den


def next_eta(eta: float, s, beta: float) -> float:
    if s is None:
        return eta
    rel = min(max(s / ALPHA / eta - 1.0, -1.0), 1.0)
    return min(eta * float(np.exp(min(GAMMA * eta, beta) * rel)), 1.0)


def lra_step(lra: LraState, dm_loc, dS_loc) -> float:
    """Items 3 and 4 on the local differences Δ̃m and Δ̃Σ (already divided by √2).  Returns η_m before the update."""
    lra.E_mean = (1.0 - BETA_MEAN) * lra.E_mean + BETA_MEAN * dm_loc
    lra.E_Sigma = (1.0 - BETA_SIGMA) * lra.E_Sigma + BETA_SIGMA * dS_loc
    lra.V_mean = (1.0 - BETA_MEAN) * lra.V_mean + BETA_MEAN * float((dm_loc ** 2).sum())
    lra.V_Sigma = (1.0 - BETA_SIGMA) * lra.V_Sigma + BETA_SIGMA * float((dS_loc ** 2).sum())
    before = lra.eta_mean
    lra.eta_mean = next_eta(lra.eta_mean, snr(float((lra.E_mean ** 2).sum()), lra.V_mean, BETA_MEAN), BETA_MEAN)
    lra.eta_Sigma = next_eta(lra.eta_Sigma, snr(float((lra.E_Sigma ** 2).sum()), lra.V_Sigma, BETA_SIGMA), BETA_SIGMA)
    return before


def lra_tell(state: O.CmaState, lra: LraState, Y, fitness, **kw) -> O.CmaState:
    """``cma_oracle.tell`` (``kw`` passed on: znorm2, h_sigma), then items 2–5."""
    m0, s0, C0 = state.mean.copy(), state.sigma, state.C.copy()
    B, d = O.eigen(C0)
    P = (B / d) @ B.T / s0
    O.tell(state, Y, fitness, **kw)
    s1 = state.sigma
    dm = state.mean - m0
    Sigma0 = s0 * s0 * C0
    dS = s1 * s1 * state.C - Sigma0
    before = lra_step(lra, P @ dm, P @ dS @ P / np.sqrt(2.0))
    state.mean = m0 + lra.eta_mean * dm
    Sigma = Sigma0 + lra.eta_Sigma * dS
    ev = np.linalg.eigvalsh((Sigma + Sigma.T) / 2 / (s1 * s1))
    ev = np.where(ev <= 0, O.EPS, ev)
    sigma = min(s1 * float(np.exp(np.log(ev).sum() / (2.0 * len(ev)))), SIGMA_MAX)
    state.C = Sigma / (sigma * sigma)
    state.sigma = sigma * before / lra.eta_mean
    return state
