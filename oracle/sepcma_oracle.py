"""CPU oracle for separable CMA-ES (sep-CMA-ES; R. Ros, N. Hansen, "A Simple Modification in CMA-ES Achieving Linear Time
and Space Complexity", PPSN 2008), as CyberAgent's ``cmaes`` library implements it (``SepCMA``) and Optuna's
``CmaEsSampler(use_separable_cma=True)`` uses it: Katib ``cmaes`` with ``use_separable_cma: true``.  Builds on
``cma_oracle`` (χ_n, the objectives, ``EPS``) and ``cma_restart_oracle`` (the history ring, tolx, term), and leaves them
unchanged.

TEST INFRASTRUCTURE ONLY, FP64 NumPy.  PARITY UNPINNED: neither ``cmaes`` nor Optuna is available offline, so every rule
below is written from memory and marked [RECALL]; where memory and the paper disagree, the paper wins.

C is restricted to its diagonal (a vector here), so sampling and update are O(D) per sample.
1. Weights [RECALL]: positive only, w_i ∝ ln((λ+1)/2) − ln i for i ≤ μ = ⌊λ/2⌋, normalised to sum to 1;
   μ_eff = 1/Σ w_i².  No active (negative) weights, unlike ``cma_oracle``.
2. Learning rates [RECALL]: c1 = 2/((D+1.3)² + μ_eff);
   cμ = (D+2)/3 · [2/μ_eff/(D+√2)² + (1 − 1/μ_eff)·min(1, (2μ_eff − 1)/((D+2)² + μ_eff))] (the paper's c_cov scaled by
   (D+2)/3); c_c = 4/(D+4); c_σ, d_σ, χ_n and c_m = 1 as in ``cma_oracle.CmaParams``.
3. Sampling [RECALL]: d = √C elementwise, y = d∘z, x = m + σ·y.
4. Tell [RECALL], in the order the samples were drawn, ranked as ``cma_oracle.tell`` ranks them:
   y_w = Σ_{i≤μ} w_i y_{i:λ}; m ← m + c_m·σ·y_w;
   p_σ ← (1 − c_σ)·p_σ + √(c_σ(2 − c_σ)μ_eff)·y_w/d, with d from before the tell;
   σ ← σ·exp((c_σ/d_σ)(‖p_σ‖/χ_n − 1)), capped at 1e32; h_σ as in ``cma_oracle.tell``;
   p_c ← (1 − c_c)·p_c + h_σ·√(c_c(2 − c_c)μ_eff)·y_w;
   C ← (1 + c1·δ(h_σ) − c1 − cμ)·C + c1·p_c² + cμ·Σ_{i≤μ} w_i y_{i:λ}², δ(h_σ) = (1 − h_σ)·c_c(2 − c_c).
5. Termination test [RECALL]: ``cma_restart_oracle.should_stop``'s criteria without NOEFFECTAXIS: TOLFUN over the same ring
   of 2·term best/worst values; TOLX: all σ·C_j < tolx and all σ·p_c,j < tolx (σ·C_j, not σ·√C_j, as the full test takes
   σ·C_ii); TOLXUP: σ·max d > 1e4; NOEFFECTCOORD: any m_j == m_j + (0.2σ)·√C_j; CONDITIONCOV: max d/min d > 1e14.

Stated departures:
(a) d = √C takes C_j ≤ 0 as ``EPS``, where upstream replaces only C_j < 0; an exact zero would divide by zero in y_w/d.
    ``cma_oracle.eigen`` makes the same departure for the same reason.
(b) cμ is capped at 1 − c1 − 1e-8, as ``cma_oracle.CmaParams`` caps the full path's.  The recalled formula exceeds 1 at
    large populations (about 5.0 at D = 128, λ = 4096, and 4.0 at D = 10, λ = 4096): C's own coefficient
    1 − c1 − cμ is then negative, C_j turns negative within three generations and the run ends in NaN.  With the
    default population 4 + ⌊3 ln D⌋ the cap never binds for D ≥ 2.

As in the other ``cmaes`` oracles, the service's own conventions hold: the search runs in the cube [0, 1]^D and a sample is
clipped into it for the trial, while the step y that the tell ranks is the unclipped one, so the oracle never sees a clip.
"""
from __future__ import annotations

import numpy as np

from . import cma_oracle as O
from . import cma_restart_oracle as R

SIGMA_MAX = 1e32
MAX_D = 4096


class SepParams:
    """Strategy parameters for dimension n and population λ (items 1 and 2)."""

    def __init__(self, n: int, popsize: int):
        assert n >= 1 and popsize >= 2
        self.n, self.popsize = n, popsize
        mu = popsize // 2
        wp = np.log((popsize + 1) / 2.0) - np.log(np.arange(1, mu + 1))
        self.weights = wp / wp.sum()
        self.mu = mu
        self.mu_eff = mu_eff = 1.0 / float((self.weights ** 2).sum())
        self.cm = 1.0
        self.c_sigma = (mu_eff + 2) / (n + mu_eff + 5)
        self.d_sigma = 1 + 2 * max(0.0, np.sqrt((mu_eff - 1) / (n + 1)) - 1) + self.c_sigma
        self.cc = 4.0 / (n + 4.0)
        self.c1 = 2.0 / ((n + 1.3) ** 2 + mu_eff)
        cmu = (n + 2) / 3.0 * (2.0 / mu_eff / (n + np.sqrt(2.0)) ** 2
                               + (1 - 1 / mu_eff) * min(1.0, (2 * mu_eff - 1) / ((n + 2) ** 2 + mu_eff)))
        self.cmu = min(1 - self.c1 - 1e-8, cmu)                  # departure (b)
        self.chi_n = np.sqrt(n) * (1.0 - 1.0 / (4.0 * n) + 1.0 / (21.0 * n * n))


class SepState:
    def __init__(self, mean, sigma, popsize):
        self.mean = np.asarray(mean, dtype=np.float64).copy()
        n = len(self.mean)
        self.p = SepParams(n, popsize)
        self.sigma = float(sigma)
        self.C = np.ones(n)
        self.p_sigma = np.zeros(n)
        self.pc = np.zeros(n)
        self.g = 0


def sqrt_c(C):
    """d = √C with C_j ≤ 0 taken as EPS (the stated departure)."""
    C = np.asarray(C, dtype=np.float64)
    return np.sqrt(np.where(C <= 0, O.EPS, C))


def ask(state: SepState, z):
    """x_k = m + σ·(d∘z_k) for the supplied standard normals z (λ×n).  Returns (X, Y)."""
    Y = np.asarray(z, dtype=np.float64) * sqrt_c(state.C)
    return state.mean + state.sigma * Y, Y


def h_left(state: SepState, norm_ps: float) -> float:
    return norm_ps / np.sqrt(1 - (1 - state.p.c_sigma) ** (2 * (state.g + 1)))


def h_threshold(p: SepParams) -> float:
    return (1.4 + 2 / (p.n + 1)) * p.chi_n


def tell(state: SepState, Y, fitness, h_sigma=None):
    """Item 4 from the steps Y = (X − m)/σ (λ×n, in sampling order) and their fitness (minimised, NumPy order, ties to the
    lower index).  ``h_sigma`` (0 or 1) overrides the stall test, for comparing with an implementation whose ‖p_σ‖ lands
    on the other side of the threshold by rounding."""
    p = state.p
    order = np.lexsort((np.arange(len(fitness)), np.asarray(fitness)))
    Ys = np.asarray(Y, dtype=np.float64)[order][:p.mu]
    d = sqrt_c(state.C)
    w = p.weights[:, None]
    y_w = (Ys * w).sum(0)
    state.mean = state.mean + p.cm * state.sigma * y_w
    state.p_sigma = (1 - p.c_sigma) * state.p_sigma + np.sqrt(p.c_sigma * (2 - p.c_sigma) * p.mu_eff) * (y_w / d)
    norm_ps = float(np.linalg.norm(state.p_sigma))
    sigma_new = min(state.sigma * float(np.exp((p.c_sigma / p.d_sigma) * (norm_ps / p.chi_n - 1))), SIGMA_MAX)
    if h_sigma is None:
        h_sigma = 1.0 if h_left(state, norm_ps) < h_threshold(p) else 0.0
    state.pc = (1 - p.cc) * state.pc + h_sigma * np.sqrt(p.cc * (2 - p.cc) * p.mu_eff) * y_w
    delta_h = (1 - h_sigma) * p.cc * (2 - p.cc)
    rank_mu = (Ys * Ys * w).sum(0)
    state.C = (1 + p.c1 * delta_h - p.c1 - p.cmu) * state.C + p.c1 * state.pc ** 2 + p.cmu * rank_mu
    state.sigma = sigma_new
    state.g += 1
    return state


def should_stop(mean, sigma, C, pc, d, hist, g: int, term: int, tol_x: float) -> int:
    """Item 5 on a state as the library stores it (C the diagonal, d = √C as stored), as a bit mask.  Bit 16
    (NOEFFECTAXIS) is never set."""
    mean, C, pc, d = (np.asarray(a, dtype=np.float64) for a in (mean, C, pc, d))
    flags = 0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if g > term and np.max(hist) - np.min(hist) < R.TOL_FUN:
            flags |= R.TOLFUN
        if np.all(sigma * C < tol_x) and np.all(sigma * pc < tol_x):
            flags |= R.TOLX
        if sigma * np.max(d) > R.TOL_XUP:
            flags |= R.TOLXUP
        if np.any(mean == mean + (0.2 * sigma) * np.sqrt(C)):
            flags |= R.NOEFFECTCOORD
        if np.max(d) / np.min(d) > R.TOL_CONDITIONCOV:
            flags |= R.CONDITIONCOV
    return flags


class Run:
    """One sep-CMA-ES run with its termination test: ``SepState`` plus the history ring."""

    def __init__(self, mean, sigma0, popsize):
        self.state = SepState(mean, sigma0, popsize)
        self.term = R.funhist_term(len(self.state.mean), popsize)
        self.tolx = R.tolx(sigma0)
        self.hist = np.zeros(2 * self.term)

    def tell(self, Y, fitness, **kw) -> int:
        s = tell(self.state, Y, fitness, **kw)
        R.record(self.hist, s.g, self.term, fitness)
        return should_stop(s.mean, s.sigma, s.C, s.pc, sqrt_c(s.C), self.hist, s.g, self.term, self.tolx)
