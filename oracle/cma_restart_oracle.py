"""CPU oracle for CMA-ES restarts (Katib ``cmaes`` with ``restart_strategy`` ``ipop`` / ``bipop``): the termination test
that triggers a restart and the IPOP / BIPOP schedules that choose the next run.  Builds on ``cma_oracle.CmaState`` /
``tell`` and leaves them unchanged.

TEST INFRASTRUCTURE; the schedule code is the service's own (``kubeflow_b200/suggestion/cma_restart.py``, re-exported
here), so the oracle and the service make the same draws.  PARITY UNPINNED: neither goptuna nor CyberAgent's ``cmaes`` (which goptuna
ports) is available offline, so what is taken from them is written from memory and marked [RECALL].

Termination test — ``cmaes``' ``CMA.should_stop`` [RECALL], evaluated after each tell on the updated state; g is the
strategy generation after the increment, n = D, d the square roots of the eigenvalues as the library stores them, c = diag(C):
  tolx = 1e-12·σ0 (σ0 of this run), tolxup = 1e4, tolfun = 1e-12, tolconditioncov = 1e14, term = 10 + ⌈30·n/λ⌉;
  history: slot 2·(g mod term) gets the generation's best fitness, slot +1 its worst (NumPy order: NaN if any is NaN);
  TOLFUN        g > term and max(hist) − min(hist) < tolfun (NaN anywhere, or inf − inf, gives False)
  TOLX          all(σ·c < tolx) and all(σ·p_c < tolx)   (p_c signed, as recalled)
  TOLXUP        σ·max(d) > tolxup
  NOEFFECTCOORD any(m == m + (0.2·σ)·√c)
  NOEFFECTAXIS  all(m == m + ((0.1·σ)·d_i)·B[:, i]), i = g mod n
  CONDITIONCOV  max(d)/min(d) > tolconditioncov
``cmaes`` stops at the first criterion that holds; here each sets its own bit.  One departure: ``cmaes`` takes the
eigenpairs in ``eigh``'s ascending order, the library its warm-started Jacobi basis; column i is whatever B's column i is.

Schedules (restarts only after a fully told generation; each run starts at C = I, zero paths, strategy generation 0, a mean
drawn uniformly in [0, 1]^D as in Auger & Hansen 2005 and Optuna's sampler — goptuna's choice is [RECALL]):
  IPOP   λ_k = λ0·2^k, σ0 unchanged.
  BIPOP  (Hansen 2009) run 0 is large; a finished run adds λ·g to its regime's budget; if budget_small < budget_large the
         next run is small, λ = ⌊λ0·(½·λ_large/λ0)^{U1²}⌋, σ = σ0·10^{−2·U2}; else it is large, i_large += 1,
         λ_large = λ0·2^{i_large}, σ = σ0.
Draws for restart k: a NumPy Generator seeded with (random_state, k); the mean first, then U1 and U2 (BIPOP only).
Every λ is clamped to [4, 8192], the limits of ``kbo_cma_create`` (a departure: upstream has no cap, and its small runs
may go below 4).
"""
from __future__ import annotations

import math

import numpy as np

from kubeflow_b200.suggestion.cma_restart import (LAMBDA_MAX, LAMBDA_MIN, STRATEGIES, Schedule, clamp,  # noqa: F401
                                                  default_popsize, restart_draws)

from . import cma_oracle as O

TOLFUN, TOLX, TOLXUP, NOEFFECTCOORD, NOEFFECTAXIS, CONDITIONCOV = 1, 2, 4, 8, 16, 32
BITS = dict(TOLFUN=TOLFUN, TOLX=TOLX, TOLXUP=TOLXUP, NOEFFECTCOORD=NOEFFECTCOORD, NOEFFECTAXIS=NOEFFECTAXIS,
            CONDITIONCOV=CONDITIONCOV)
TOL_XUP, TOL_FUN, TOL_CONDITIONCOV = 1e4, 1e-12, 1e14


def funhist_term(n: int, popsize: int) -> int:
    return 10 + math.ceil(30 * n / popsize)


def tolx(sigma0: float) -> float:
    return 1e-12 * sigma0


def record(hist, g: int, term: int, fitness):
    """Write generation g's best and worst fitness (NumPy sort order, NaN last) into the ring ``hist`` (2·term)."""
    f = np.sort(np.asarray(fitness, dtype=np.float64))
    i = 2 * (g % term)
    hist[i], hist[i + 1] = f[0], f[-1]
    return hist


def should_stop(mean, sigma, C, pc, B, d, hist, g: int, term: int, tol_x: float) -> int:
    """The six criteria on a state as the library stores it, as a bit mask (every criterion evaluated)."""
    mean, pc, d, B = (np.asarray(a, dtype=np.float64) for a in (mean, pc, d, B))
    c = np.diag(np.asarray(C, dtype=np.float64))
    n = len(mean)
    flags = 0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if g > term and np.max(hist) - np.min(hist) < TOL_FUN:
            flags |= TOLFUN
        if np.all(sigma * c < tol_x) and np.all(sigma * pc < tol_x):
            flags |= TOLX
        if sigma * np.max(d) > TOL_XUP:
            flags |= TOLXUP
        if np.any(mean == mean + (0.2 * sigma) * np.sqrt(c)):
            flags |= NOEFFECTCOORD
        i = g % n
        if np.all(mean == mean + ((0.1 * sigma) * d[i]) * B[:, i]):
            flags |= NOEFFECTAXIS
        if np.max(d) / np.min(d) > TOL_CONDITIONCOV:
            flags |= CONDITIONCOV
    return flags


class Run:
    """One CMA-ES run of the oracle with its termination test: ``cma_oracle.CmaState`` plus the history ring."""

    def __init__(self, mean, sigma0, popsize):
        self.state = O.CmaState(mean, sigma0, popsize)
        self.term = funhist_term(len(self.state.mean), popsize)
        self.tolx = tolx(sigma0)
        self.hist = np.zeros(2 * self.term)

    def tell(self, Y, fitness, **kw) -> int:
        """``cma_oracle.tell``, then the history and the criteria on the updated state (eigenpairs from ``eigh``)."""
        s = O.tell(self.state, Y, fitness, **kw)
        record(self.hist, s.g, self.term, fitness)
        B, d = O.eigen(s.C)
        return should_stop(s.mean, s.sigma, s.C, s.pc, B, d, self.hist, s.g, self.term, self.tolx)
