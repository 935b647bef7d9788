"""Request conversion — the host-side mirror of kubeflow/katib ``pkg/suggestion/v1beta1/internal/``
(``search_space.py``: HyperParameterSearchSpace / HyperParameter; ``trial.py``: Trial / Assignment / Metric;
``constant.py``).  Same names and argument meaning so the tests read like upstream's (SURVEY.md §8(a) A1/A2).
All numeric values travel as strings on the wire."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import api_pb as api

INTEGER, DOUBLE, CATEGORICAL, DISCRETE = "int", "double", "categorical", "discrete"
MAX_GOAL, MIN_GOAL = "MAXIMIZE", "MINIMIZE"


class AlgorithmSettingsError(ValueError):
    """Raised for anything ValidateAlgorithmSettings / conversion rejects → gRPC INVALID_ARGUMENT."""


@dataclass
class HyperParameter:
    name: str
    type: str
    min: str | None = None
    max: str | None = None
    list: list = field(default_factory=list)
    step: str | None = None

    @staticmethod
    def int(name, min_, max_, step=None):
        return HyperParameter(name, INTEGER, min_, max_, [], step)

    @staticmethod
    def double(name, min_, max_, step=None):
        return HyperParameter(name, DOUBLE, min_, max_, [], step)

    @staticmethod
    def categorical(name, lst):
        return HyperParameter(name, CATEGORICAL, None, None, list(lst))

    @staticmethod
    def discrete(name, lst):
        return HyperParameter(name, DISCRETE, None, None, list(lst))


@dataclass
class HyperParameterSearchSpace:
    goal: str
    params: list

    @staticmethod
    def convert(experiment) -> "HyperParameterSearchSpace":
        t = experiment.spec.objective.type
        if t == api.MAXIMIZE:
            goal = MAX_GOAL
        elif t == api.MINIMIZE:
            goal = MIN_GOAL
        else:
            raise AlgorithmSettingsError("objective.type must be MINIMIZE or MAXIMIZE")
        params = []
        for p in experiment.spec.parameter_specs.parameters:
            fs = p.feasible_space
            if p.parameter_type == api.INT:
                hp = HyperParameter.int(p.name, fs.min, fs.max, fs.step or None)
            elif p.parameter_type == api.DOUBLE:
                hp = HyperParameter.double(p.name, fs.min, fs.max, fs.step or None)
            elif p.parameter_type == api.CATEGORICAL:
                hp = HyperParameter.categorical(p.name, fs.list)
            elif p.parameter_type == api.DISCRETE:
                hp = HyperParameter.discrete(p.name, fs.list)
            else:
                raise AlgorithmSettingsError(f"parameter {p.name!r}: unknown parameter_type {p.parameter_type}")
            params.append(hp)
        if not params:
            raise AlgorithmSettingsError("experiment has no parameters")
        for hp in params:
            if hp.type in (INTEGER, DOUBLE):
                try:
                    lo, hi = float(hp.min), float(hp.max)
                except (TypeError, ValueError):
                    raise AlgorithmSettingsError(f"parameter {hp.name!r}: min/max must be numbers, got {hp.min!r}/{hp.max!r}")
                if not lo < hi:
                    raise AlgorithmSettingsError(f"parameter {hp.name!r}: need min < max, got {hp.min} >= {hp.max}")
            elif not hp.list:
                raise AlgorithmSettingsError(f"parameter {hp.name!r}: empty feasible list")
        return HyperParameterSearchSpace(goal, params)


@dataclass
class Assignment:
    name: str
    value: str

    @staticmethod
    def convert(assignments):
        return [Assignment(a.name, a.value) for a in assignments]


@dataclass
class Metric:
    name: str
    value: str


@dataclass
class Trial:
    name: str
    assignments: list
    target_metric: Metric
    metric_name: str
    additional_metrics: list

    @staticmethod
    def convert(trials, skip_names=None):
        """Only trials that finished with an observation of the objective metric are usable (upstream: succeeded trials).
        ``skip_names``: names already consumed by the caller — Katib resends EVERY finished trial on every call, so at
        N = 8192 trials × 32 parameters building Python objects for all of them costs ~0.3 s per request; skipping the known
        ones by name keeps a steady-state request at the cost of one attribute read per trial (SURVEY.md §8(f)3)."""
        out = []
        for t in trials:
            if skip_names is not None and t.name in skip_names:
                continue
            if t.status.condition not in (api.SUCCEEDED, api.EARLYSTOPPED):
                continue
            name = t.spec.objective.objective_metric_name
            target, extra = None, []
            for m in t.status.observation.metrics:
                if m.name == name or (not name and target is None):
                    target = Metric(m.name, m.value)
                else:
                    extra.append(Metric(m.name, m.value))
            if target is None:
                continue
            out.append(Trial(t.name, Assignment.convert(t.spec.parameter_assignments.assignments), target, name, extra))
        return out


def parse_settings(experiment) -> dict:
    return {s.name: s.value for s in experiment.spec.algorithm.algorithm_settings}


def spec_values(p, where: str, limit: int) -> list:
    """The values of one ``ParameterSpec``, in order [RECALL: Katib's ENAS Operation.py and its Optuna service's grid search]:
    INT → range(min, max + 1, step), DOUBLE → np.arange(min, max + step, step) with an endpoint above max dropped,
    CATEGORICAL and DISCRETE → the feasible list as strings.  AlgorithmSettingsError, prefixed by ``where``, for a spec with no
    such values or with more than ``limit`` of them (checked before any list is built)."""
    fs = p.feasible_space
    if p.parameter_type in (api.CATEGORICAL, api.DISCRETE):
        if not len(fs.list):
            kind = "CATEGORICAL" if p.parameter_type == api.CATEGORICAL else "DISCRETE"
            raise AlgorithmSettingsError(f"{where}: a {kind} spec needs a non-empty list")
        return [str(x) for x in fs.list]
    if p.parameter_type not in (api.INT, api.DOUBLE):
        raise AlgorithmSettingsError(f"{where}: only INT, DOUBLE, CATEGORICAL and DISCRETE specs have values")
    if not (fs.min and fs.max and fs.step):
        raise AlgorithmSettingsError(f"{where}: INT and DOUBLE specs need min, max and step")
    try:
        if p.parameter_type == api.INT:
            lo, hi, st = int(fs.min), int(fs.max), int(fs.step)
        else:
            lo, hi, st = float(fs.min), float(fs.max), float(fs.step)
    except ValueError:
        raise AlgorithmSettingsError(f"{where}: min, max and step must be numbers")
    if not (st > 0 and lo <= hi and np.isfinite(lo) and np.isfinite(hi) and np.isfinite(st)):
        raise AlgorithmSettingsError(f"{where}: need step > 0 and min <= max")
    if (hi - lo) / st >= limit:
        raise AlgorithmSettingsError(f"{where}: more than this engine's limit of {limit} values")
    if p.parameter_type == api.INT:
        return list(range(lo, hi + 1, st))
    vals = np.arange(lo, hi + st, st)
    if vals[-1] > hi:
        vals = vals[:-1]
    return [float(x) for x in vals]
