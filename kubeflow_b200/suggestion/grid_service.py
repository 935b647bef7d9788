"""``grid`` — Katib's grid search, which upstream serves from its Optuna image through ``optuna.samplers.GridSampler``.  Neither
Katib's service nor Optuna is at hand; their rules are restated from memory and marked [RECALL].

This is host-side bookkeeping by nature (a mixed-radix decode per point and a set of visited ids); there is nothing for the GPU
to do here and none is used.

* Grid [RECALL: Katib's Optuna service]: each parameter's values by ``internal.spec_values``: INT → range(min, max + 1, step),
  step 1 when unset; DOUBLE → np.arange(min, max + step, step) with an endpoint above max dropped; CATEGORICAL and DISCRETE →
  the feasible list in its order.
* Points [RECALL: GridSampler]: the Cartesian product over the parameters sorted by name, the last name varying fastest
  (``itertools.product`` over the sorted search space).  Point id i is i written in that mixed radix, so no list of points is
  ever built.  A reply lists each point's values in the Experiment's parameter order, formatted as ``BaseSkoptService.convert``.
* ValidateAlgorithmSettings: a DOUBLE parameter needs step > 0 and an INT step must be > 0 [RECALL]; ``max_trial_count`` > 0 may
  not exceed the number of points, and the message names both [RECALL]; the one setting is ``random_state``, an integer >= 0.
* Visited, recomputed on every call: every trial of ``request.trials`` whatever its condition, matched to a point by its
  assigned values (INT and DOUBLE compared as numbers, CATEGORICAL and DISCRETE as strings; a trial matching no point is
  ignored), plus the ids this process issued for the experiment that have not come back as trials yet.  So a restarted service
  never re-issues a point Katib already has.
* Draw [RECALL: GridSampler]: each point is drawn uniformly from the ids neither finished (SUCCEEDED, EARLYSTOPPED, FAILED,
  KILLED, METRICSUNAVAILABLE) nor in flight (any other condition, or issued and not back); when there is none, from the ids
  not finished; when every id has finished, from all ids (a point is then evaluated again, and logged).  The points of one
  call are drawn in turn, each in flight for the next.

Departures, all deliberate:
* the draws come from a NumPy Generator seeded by ``random_state`` (fresh entropy without it), kept per experiment: the same
  requests give the same points, but not the points Optuna's RandomState stream would give;
* this engine refuses, by name, a parameter with more than ``MAX_VALUES`` values, a grid of more than ``MAX_POINTS`` points
  (so every id and count fits in an int64) and two parameters of the same name.
"""
from __future__ import annotations

import bisect
import logging
import math

import numpy as np

from . import api_pb as api
from .internal import AlgorithmSettingsError, HyperParameterSearchSpace, parse_settings, spec_values
from .service import _Base, _reply_from, experiment_fingerprint

logger = logging.getLogger(__name__)

NAME = "grid"
MAX_VALUES = 1 << 20          # values of one parameter: each parameter's list is built
MAX_POINTS = 1 << 62          # points of the grid: ids are never materialised, only counted
_FINISHED = (api.SUCCEEDED, api.EARLYSTOPPED, api.FAILED, api.KILLED, api.METRICSUNAVAILABLE)


def validate_grid_settings(settings: dict) -> dict:
    out = {}
    for k, v in settings.items():
        if k != "random_state":
            raise AlgorithmSettingsError(f"unknown setting {k} for algorithm {NAME}")
        try:
            out[k] = int(v)
        except ValueError:
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
        if out[k] < 0:
            raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")
    return out


class Grid:
    """The grid of one Experiment's ``parameter_specs``: per parameter (in Experiment order) its values, and point ids in the
    mixed radix of the parameters sorted by name."""

    def __init__(self, specs):
        self.values = []
        for p in specs:
            where = f"parameter {p.name!r}"
            if p.parameter_type == api.DOUBLE and not p.feasible_space.step:
                raise AlgorithmSettingsError(f"{where}: grid search needs a step > 0 for a DOUBLE parameter")
            if p.parameter_type == api.INT and not p.feasible_space.step:
                q = api.ParameterSpec()
                q.CopyFrom(p)
                q.feasible_space.step = "1"
                p = q
            self.values.append(spec_values(p, where, MAX_VALUES))
        self.names = [p.name for p in specs]
        if len(set(self.names)) != len(self.names):
            dup = sorted(n for n in set(self.names) if self.names.count(n) > 1)
            raise AlgorithmSettingsError(f"parameter names must be unique for grid search: {dup} appear more than once")
        self.order = sorted(range(len(specs)), key=lambda j: self.names[j])     # most significant digit first
        self.size = math.prod(len(v) for v in self.values)
        if self.size > MAX_POINTS:
            raise AlgorithmSettingsError(f"the grid has {self.size} points, more than this engine's limit of {MAX_POINTS} points")
        self._parse = [int if p.parameter_type == api.INT else float if p.parameter_type == api.DOUBLE else None for p in specs]
        self._index = [None if parse else {s: i for i, s in reversed(list(enumerate(v)))} for v, parse in zip(self.values, self._parse)]

    def point(self, i: int) -> list:
        """The values of point ``i``, in Experiment order."""
        out = [None] * len(self.values)
        for j in reversed(self.order):
            i, d = divmod(i, len(self.values[j]))
            out[j] = self.values[j][d]
        return out

    def _digit(self, j: int, text: str):
        if self._parse[j] is None:
            return self._index[j].get(text)
        try:
            x = self._parse[j](text)
        except ValueError:
            return None
        d = bisect.bisect_left(self.values[j], x)          # INT and DOUBLE values ascend: step > 0
        return d if d < len(self.values[j]) and self.values[j][d] == x else None

    def id_of(self, assignments) -> int | None:
        """The id of the point whose values ``assignments`` (ParameterAssignment messages) carry, or None when they match none."""
        by_name = {a.name: a.value for a in assignments}
        i = 0
        for j in self.order:
            text = by_name.get(self.names[j])
            d = None if text is None else self._digit(j, text)
            if d is None:
                return None
            i = i * len(self.values[j]) + d
        return i


def check_experiment(experiment) -> tuple:
    """(search space, settings, Grid), or AlgorithmSettingsError naming the parameter or setting."""
    ss = HyperParameterSearchSpace.convert(experiment)
    settings = validate_grid_settings(parse_settings(experiment))
    grid = Grid(experiment.spec.parameter_specs.parameters)
    m = int(experiment.spec.max_trial_count)
    if m > grid.size:
        raise AlgorithmSettingsError(f"Max Trial Count: {m} > all possible search space combinations: {grid.size}")
    return ss, settings, grid


def _nth_free(r: int, excluded: list) -> int:
    """The r-th id (from 0) not in ``excluded`` (ascending, distinct)."""
    for e in excluded:
        if e > r:
            break
        r += 1
    return r


def draw(grid_size: int, finished: set, in_flight: set, rng, k: int) -> list:
    """k ids, each uniform over the ids neither finished nor in flight, else over the ids not finished, else over all ids;
    each id drawn is in flight for the next draw."""
    busy, done = sorted(finished | in_flight), sorted(finished)
    out = []
    for _ in range(k):
        excluded = busy if len(busy) < grid_size else done if len(done) < grid_size else []
        i = _nth_free(int(rng.integers(grid_size - len(excluded))), excluded)
        j = bisect.bisect_left(busy, i)
        if j == len(busy) or busy[j] != i:
            busy.insert(j, i)
        out.append(i)
    if len(done) == grid_size and k:
        logger.warning("grid: every point has finished; evaluating %d again", k)
    return out


class _GridExperiment:
    def __init__(self, random_state):
        self.rng = np.random.default_rng(random_state)
        self.issued = set()          # ids handed out and not yet seen in request.trials

    def close(self):
        pass


class GridService(_Base):
    algorithm_names = (NAME,)
    MAX_EXPERIMENTS = 64          # an entry is a Generator and a set of ids, no device memory

    def validate(self, experiment):
        self.check_algorithm(experiment)
        check_experiment(experiment)

    def get_suggestions(self, request):
        from .base_service import BaseSkoptService
        exp = request.experiment
        self.check_algorithm(exp)
        ss, settings, grid = check_experiment(exp)
        k = max(int(request.current_request_number), 0)
        if k == 0:
            return _reply_from([])
        finished, running = set(), set()
        for t in request.trials:
            i = grid.id_of(t.spec.parameter_assignments.assignments)
            if i is not None:
                (finished if t.status.condition in _FINISHED else running).add(i)
        with self._lock:
            entry = self.experiment(exp.name, experiment_fingerprint(exp, ss, settings),
                                    lambda: _GridExperiment(settings.get("random_state")))
            entry.issued -= finished | running
            in_flight = running | entry.issued
            ids = draw(grid.size, finished, in_flight, entry.rng, k)
            entry.issued.update(ids)
        logger.info("grid %s: %d of %d points finished, %d in flight before this call, %d issued", exp.name, len(finished),
                    grid.size, len(in_flight), len(ids))
        return _reply_from([BaseSkoptService.convert(ss, grid.point(i)) for i in ids])
