"""CPU oracle for CMA-ES with Margin (CMAwM; R. Hamano, S. Saito, M. Nomura, S. Shirakawa, "CMA-ES with Margin:
Lower-Bounding Marginal Probability for Mixed-Integer Black-Box Optimization", GECCO 2022), as CyberAgent's ``cmaes``
library implements it and Optuna's ``CmaEsSampler(with_margin=True)`` uses it: Katib ``cmaes`` with ``with_margin: true``.
Builds on ``cma_oracle.CmaState`` / ``tell`` and leaves them unchanged.

TEST INFRASTRUCTURE ONLY, FP64 NumPy / SciPy.  PARITY UNPINNED: neither ``cmaes`` nor the paper is available offline, so
every rule taken from them is written from memory and marked [RECALL].

1. Coordinates [RECALL for the thresholds]: the search stays in the service's cube [0, 1]^D.  A discrete dimension j has
   sorted levels v_1 < … < v_K in cube coordinates — a table, or first + k·step for integer ranges too long for one —
   and thresholds ℓ_k = (v_k + v_{k+1})/2.
2. Sampling [RECALL]: A is a diagonal vector, all ones at the start of a run.  y = B·(d∘z) as in ``cma_oracle.ask`` and
   x = m + σ·(A∘y).  A discrete coordinate encodes to the level whose interval (ℓ_{k−1}, ℓ_k] holds x_j (v_1 below ℓ_1,
   v_K above ℓ_{K−1}).  The trial gets the encoded value; the update uses y.  (Continuous coordinates are clipped to the
   cube by the service, as without the margin; ``cmaes`` resamples them instead.)
3. Update [RECALL]: ``cma_oracle.tell`` on y, except that the mean step is m ← m + c_m·σ·A∘Σ w_i y_{i:λ}.
4. Margin correction [RECALL], after the update, for each discrete dimension j, with s_j = σ·A_j·√C_jj and the interval
   ℓ_lo ≤ m_j < ℓ_up of m_j (both limits are the one boundary threshold in the first and the last interval):
     p_lo = Φ((ℓ_lo − m_j)/s_j), p_up = Φ((m_j − ℓ_up)/s_j), p_mid = 1 − p_lo − p_up.
   Edge case, max(p_lo, p_up) > 0.5: if min(p_lo, p_up) < α, m_j ← ℓ_up + sign(m_j − ℓ_up)·s_j·Φ⁻¹(1 − α).
   Side case, max(p_lo, p_up) ≤ 0.5: p_lo, p_up ← max(·, α/2); each takes its share of the overshoot,
     p'_lo = p_lo + (1 − p_lo − p_up − p_mid)·(p_lo − α/2)/(p_lo + p_mid + p_up − 3α/2) (same for p_up), clipped to
     [1e-10, 0.5 − 1e-10]; with χ = Φ⁻¹(1 − p'), A_j ← (ℓ_up − ℓ_lo)/((χ_lo + χ_up)·σ·√C_jj) and
     m_j ← (ℓ_lo·χ_up + ℓ_up·χ_lo)/(χ_lo + χ_up), σ and C fixed.
   Upstream writes p_up as 1 − Φ((ℓ_up − m_j)/s_j) and Φ⁻¹(1 − p) as √χ²₁.ppf(1 − 2p); both lose the small tail to
   cancellation (an absolute 1e-16 on a tail of α/2 ≈ 1e-6), so this file takes the same quantities from the tails
   themselves: Φ by ``scipy.special.ndtr`` and Φ⁻¹(1 − p) as √χ²₁.isf(2p).
5. α defaults to 1/(D·λ) [RECALL], recomputed for the λ of every IPOP / BIPOP run, and a restart resets A to ones.
The termination test reads the inner state (m, σ, C, paths) as without the margin.
"""
from __future__ import annotations

import numpy as np
from scipy.special import ndtr
from scipy.stats import chi2

from . import cma_oracle as O

CLIP = 1e-10


def default_alpha(D: int, popsize: int) -> float:
    return 1.0 / (D * popsize)


def level(dim, k):
    """v_k (0-based) of a discrete dimension: a sorted table (array) or (first, step, count)."""
    k = np.asarray(k)
    if isinstance(dim, tuple):
        return dim[0] + k.astype(np.float64) * dim[1]
    return np.asarray(dim, dtype=np.float64)[k]


def count(dim) -> int:
    return int(dim[2]) if isinstance(dim, tuple) else len(dim)


def threshold(dim, k):
    return (level(dim, k) + level(dim, np.asarray(k) + 1)) * 0.5


def rank(dim, x, inclusive: bool):
    """Number of thresholds ℓ_k < x (or ≤ x with ``inclusive``), by a vectorised binary search over k < count − 1."""
    x = np.asarray(x, dtype=np.float64)
    lo = np.zeros(x.shape, dtype=np.int64)
    hi = np.full(x.shape, count(dim) - 1, dtype=np.int64)
    while np.any(lo < hi):
        act = lo < hi
        mid = lo + ((hi - lo) >> 1)
        l = threshold(dim, np.where(act, mid, 0))
        go = (l <= x) if inclusive else (l < x)
        lo = np.where(act & go, mid + 1, lo)
        hi = np.where(act & ~go, mid, hi)
    return lo


def encode(dims: dict, X):
    """Each discrete coordinate to the level whose interval (ℓ_{k−1}, ℓ_k] holds it; continuous ones unchanged."""
    X = np.array(X, dtype=np.float64, copy=True)
    for j, dim in dims.items():
        X[..., j] = level(dim, rank(dim, X[..., j], inclusive=False))
    return X


def limits(dim, m):
    """(ℓ_lo, ℓ_up) of the interval ℓ_lo ≤ m < ℓ_up; the boundary threshold twice in the first and last interval."""
    r = int(rank(dim, m, inclusive=True))
    K = count(dim)
    return float(threshold(dim, 0 if r == 0 else r - 1)), float(threshold(dim, r - 1 if r == K - 1 else r))


def tails(m, s, l_lo, l_up):
    p_lo = float(ndtr((l_lo - m) / s))
    p_up = float(ndtr((m - l_up) / s))
    return p_lo, p_up


def chi_upper(p):
    """Φ⁻¹(1 − p) = √χ²₁.ppf(1 − 2p), taken as √χ²₁.isf(2p)."""
    return float(np.sqrt(chi2.isf(2.0 * p, df=1)))


def margin_step(mean, A, sigma, c_diag, dims: dict, alpha: float, info: dict | None = None):
    """Item 4 on (m, A) after the update.  Returns (m, A, cases) with cases[j] in {"edge", "edge-moved", "side"}.
    ``info``, if given, receives {j: (q_lo, q_up, χ_lo, χ_up)} for the side cases."""
    m, A = np.array(mean, dtype=np.float64), np.array(A, dtype=np.float64)
    cases = {}
    for j, dim in dims.items():
        l_lo, l_up = limits(dim, m[j])
        sc = float(np.sqrt(c_diag[j]))
        s = sigma * A[j] * sc
        p_lo, p_up = tails(m[j], s, l_lo, l_up)
        p_mid = 1.0 - p_lo - p_up
        if max(p_lo, p_up) > 0.5:
            cases[j] = "edge"
            if min(p_lo, p_up) < alpha:
                sg = float(np.sign(m[j] - l_up))
                m[j] = l_up + sg * (s * chi_upper(alpha))
                cases[j] = "edge-moved"
            continue
        cases[j] = "side"
        h = 0.5 * alpha
        lo, up = max(p_lo, h), max(p_up, h)
        over = 1.0 - lo - up - p_mid
        den = lo + p_mid + up - 3.0 * h
        q_lo = min(max(lo + over * (lo - h) / den, CLIP), 0.5 - CLIP)
        q_up = min(max(up + over * (up - h) / den, CLIP), 0.5 - CLIP)
        chi_lo, chi_up = chi_upper(q_lo), chi_upper(q_up)
        chi = chi_lo + chi_up
        if info is not None:
            info[j] = (q_lo, q_up, chi_lo, chi_up)
        A[j] = (l_up - l_lo) / (chi * sigma * sc)
        m[j] = (l_lo * chi_up + l_up * chi_lo) / chi
    return m, A, cases


def invariant_violations(mean, A, sigma, c_diag, dims: dict, alpha: float, cases: dict, before, rtol=1e-12):
    """What the margin step guarantees, checked on its result without trusting item 4's formulas: in the edge case the
    probability of crossing the boundary is at least α; in the side case each tail lies in [min(α/2, 1e-10), 0.5].
    ``before`` is the mean the step started from (its interval fixes the limits).  The bounds hold up to ``rtol`` relative
    in m_j: a tail is taken at m_j ± rtol·|m_j|, whichever favours the bound, since once s_j is small the last bit of m_j
    alone moves a tail by more than any fixed relative amount.  Returns a list of messages."""
    bad = []
    for j, dim in dims.items():
        l_lo, l_up = limits(dim, before[j])
        s = sigma * A[j] * float(np.sqrt(c_diag[j]))
        dm = rtol * max(abs(mean[j]), abs(l_lo), abs(l_up))
        (a_lo, a_up), (b_lo, b_up) = tails(mean[j] - dm, s, l_lo, l_up), tails(mean[j] + dm, s, l_lo, l_up)
        hi_lo, hi_up, lo_lo, lo_up = max(a_lo, b_lo), max(a_up, b_up), min(a_lo, b_lo), min(a_up, b_up)
        if cases[j].startswith("edge"):
            if not max(min(a_lo, a_up), min(b_lo, b_up)) >= alpha:
                bad.append(f"dim {j}: crossing probability {min(a_lo, a_up):.6g} < alpha {alpha:.6g}")
        else:
            floor = min(alpha / 2, CLIP)
            for name, hi, lo in (("lower", hi_lo, lo_lo), ("upper", hi_up, lo_up)):
                if not (hi >= floor and lo <= 0.5):
                    bad.append(f"dim {j}: {name} tail {hi:.6g} outside [{floor:.6g}, 0.5]")
    return bad


class MarginState:
    """``cma_oracle.CmaState`` plus A, the discrete dimensions and α."""

    def __init__(self, mean, sigma, popsize, dims: dict, alpha: float | None = None):
        self.state = O.CmaState(mean, sigma, popsize)
        self.dims = dict(dims)
        n = len(self.state.mean)
        self.alpha = alpha if alpha else default_alpha(n, popsize)
        self.A = np.ones(n)
        self.last_cases = {}
        self.mean_before = self.state.mean.copy()


def ask(ms: MarginState, z):
    """(encoded X, Y, unencoded x) for the supplied standard normals z (λ×n)."""
    B, D = O.eigen(ms.state.C)
    Y = (z * D) @ B.T
    X = ms.state.mean + ms.state.sigma * (ms.A * Y)
    return encode(ms.dims, X), Y, X


def tell(ms: MarginState, Y, fitness, **kw):
    """``cma_oracle.tell`` with the A-scaled mean step, then the margin correction.  With no discrete dimension this is
    ``cma_oracle.tell`` bit for bit (A = 1 multiplies exactly)."""
    s = ms.state
    m0, sigma0 = s.mean.copy(), s.sigma
    O.tell(s, Y, fitness, **kw)
    p = s.p
    order = np.lexsort((np.arange(len(fitness)), np.asarray(fitness)))
    y_w = (np.asarray(Y, dtype=np.float64)[order][:p.mu] * p.weights[:p.mu, None]).sum(0)
    s.mean = m0 + p.cm * sigma0 * (ms.A * y_w)
    ms.mean_before = s.mean.copy()
    if ms.dims:
        s.mean, ms.A, ms.last_cases = margin_step(s.mean, ms.A, s.sigma, np.diag(s.C), ms.dims, ms.alpha)
    return ms
