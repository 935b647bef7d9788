"""IPOP / BIPOP restart schedules for the ``cmaes`` service (``restart_strategy``), shared with the oracle
``oracle/cma_restart_oracle.py``, whose docstring states the contract.  Host-side NumPy: a restart makes a handful of draws."""
from __future__ import annotations

import math

import numpy as np

LAMBDA_MIN, LAMBDA_MAX = 4, 8192      # kbo_cma_create's limits
STRATEGIES = ("none", "ipop", "bipop")


def default_popsize(n: int) -> int:
    return 4 + int(3 * np.log(n))


def clamp(lam) -> int:
    return int(min(max(int(lam), LAMBDA_MIN), LAMBDA_MAX))


def restart_draws(random_state: int, k: int, n: int, bipop: bool):
    """The host draws of restart k (k = 1, 2, …): mean ~ U[0, 1]^n, then (U1, U2) for BIPOP."""
    r = np.random.default_rng([int(random_state), int(k)])
    mean = r.uniform(0.0, 1.0, n)
    u = r.uniform(0.0, 1.0, 2) if bipop else None
    return mean, u


class Schedule:
    """IPOP / BIPOP restart schedule.  ``next_run(λ, g)`` is called when a run of population λ stops after g generations
    and returns the next run's (λ, mean, σ).  ``draws`` overrides (mean, (U1, U2)) for hand-worked tests."""

    def __init__(self, strategy: str, n: int, popsize0: int | None = None, sigma0: float = 1.0 / 6.0, random_state: int = 0):
        if strategy not in ("ipop", "bipop"):
            raise ValueError(f"no restart schedule for {strategy!r}")
        self.strategy, self.n = strategy, int(n)
        self.lam0 = int(popsize0) if popsize0 else default_popsize(n)
        self.sigma0, self.random_state = float(sigma0), int(random_state)
        self.restarts = 0
        self.i_large, self.lam_large = 0, self.lam0
        self.budget = {"small": 0, "large": 0}
        self.regime = "large"
        self.history = []                               # (regime, λ, σ) of every run started by a restart

    def next_run(self, lam_run: int, gens_run: int, draws=None):
        self.restarts += 1
        mean, u = draws if draws is not None else restart_draws(self.random_state, self.restarts, self.n, self.strategy == "bipop")
        if self.strategy == "ipop":
            lam, sigma, self.regime = clamp(self.lam0 * 2 ** self.restarts), self.sigma0, "large"
        else:
            self.budget[self.regime] += int(lam_run) * int(gens_run)
            if self.budget["small"] < self.budget["large"]:
                self.regime = "small"
                lam = clamp(math.floor(self.lam0 * (0.5 * self.lam_large / self.lam0) ** (u[0] ** 2)))
                sigma = self.sigma0 * 10.0 ** (-2.0 * u[1])
            else:
                self.regime = "large"
                self.i_large += 1
                self.lam_large = self.lam0 * 2 ** self.i_large
                lam, sigma = clamp(self.lam_large), self.sigma0
        self.history.append((self.regime, lam, sigma))
        return lam, np.asarray(mean, dtype=np.float64), sigma
