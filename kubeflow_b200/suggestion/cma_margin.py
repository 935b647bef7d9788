"""Discrete dimensions of ``cmaes`` with ``with_margin: true`` (CMA-ES with Margin; oracle/cma_margin_oracle.py).

An ``int`` parameter's levels are the integers lo, lo + step, … ≤ hi (step 1 unless the feasible space gives one); a
``discrete`` parameter's are its distinct numeric values, sorted.  Both live in the search cube [0, 1] at
(v − v_first)/(v_last − v_first), as a table, or as (first, step, count) for an integer range longer than ``TABLE_MAX``
levels (a Katib ``int`` may span 2³¹).  The sampler encodes each sample to one of these cube levels; ``Levels.value``
turns it back into the trial's assignment string."""
from __future__ import annotations

import numpy as np

from .internal import DISCRETE, INTEGER, AlgorithmSettingsError

TABLE_MAX = 4096


def parse_with_margin(v, name: str = "with_margin") -> bool:
    """A boolean setting (``true`` / ``false`` in any case): ``with_margin``, or the one ``name`` gives."""
    s = str(v).strip().lower()
    if s not in ("true", "false"):
        raise AlgorithmSettingsError(f"{name} must be true or false, got {v!r}")
    return s == "true"


class Levels:
    """One discrete dimension: ``cube`` is what ``CmaEs.set_margin`` takes (a sorted array, or (first, step, count))."""

    def __init__(self, cube, strings=None, lo=0, step=1):
        self.cube, self._strings, self._lo, self._step = cube, strings, lo, step

    def index(self, u: float) -> int:
        """The level index of an encoded cube value."""
        if isinstance(self.cube, tuple):
            return int(min(max(round((u - self.cube[0]) / self.cube[1]), 0), self.cube[2] - 1))
        return int(min(np.searchsorted(self.cube, u), len(self.cube) - 1))

    def value(self, u: float) -> str:
        k = self.index(u)
        return self._strings[k] if self._strings is not None else str(self._lo + k * self._step)


def _int_levels(p) -> Levels:
    try:
        lo, hi = int(p.min), int(p.max)
        step = int(p.step) if p.step else 1
    except ValueError:
        raise AlgorithmSettingsError(f"int parameter {p.name!r}: min, max and step must be integers")
    if step < 1:
        raise AlgorithmSettingsError(f"int parameter {p.name!r}: step must be positive, got {p.step}")
    K = (hi - lo) // step + 1
    if K < 2:
        raise AlgorithmSettingsError(f"int parameter {p.name!r}: with_margin needs two or more levels")
    cstep = step / (hi - lo)
    cube = (0.0, cstep, K) if K > TABLE_MAX else np.arange(K, dtype=np.float64) * cstep
    return Levels(cube, lo=lo, step=step)


def _discrete_levels(p) -> Levels:
    try:
        vals = [float(v) for v in p.list]
    except ValueError:
        raise AlgorithmSettingsError(f"discrete parameter {p.name!r}: cmaes with_margin needs numeric values")
    if not all(np.isfinite(vals)):
        raise AlgorithmSettingsError(f"discrete parameter {p.name!r}: values must be finite")
    uniq = sorted(set(vals))
    if len(uniq) < 2:
        raise AlgorithmSettingsError(f"discrete parameter {p.name!r}: with_margin needs two or more distinct values")
    strings = [p.list[vals.index(v)] for v in uniq]
    u = np.asarray(uniq)
    return Levels((u - u[0]) / (u[-1] - u[0]), strings=strings)


def discrete_dims(params) -> dict:
    """{parameter index: Levels} of the int and discrete parameters."""
    out = {}
    for j, p in enumerate(params):
        if p.type == INTEGER:
            out[j] = _int_levels(p)
        elif p.type == DISCRETE:
            out[j] = _discrete_levels(p)
    return out


def encode(levels: dict, x):
    """x (one point in the cube, sampler coordinates) with each discrete coordinate encoded as the sampler does: to the
    level whose interval (ℓ_{k−1}, ℓ_k] of thresholds ℓ_k = (v_k + v_{k+1})/2 holds it."""
    x = np.array(x, dtype=np.float64, copy=True)
    for j, L in levels.items():
        c = L.cube
        if isinstance(c, tuple):
            first, step, K = c
            lev = lambda k: first + float(k) * step
            k = int(min(max(round((x[j] - first) / step), 0), K - 1))
            if k > 0 and x[j] <= (lev(k - 1) + lev(k)) * 0.5:
                k -= 1
            elif k < K - 1 and x[j] > (lev(k) + lev(k + 1)) * 0.5:
                k += 1
            x[j] = lev(k)
        else:
            x[j] = c[np.searchsorted((c[:-1] + c[1:]) * 0.5, x[j], side="left")]
    return x
