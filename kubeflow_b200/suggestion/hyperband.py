"""``hyperband`` — mirror of kubeflow/katib pkg/suggestion/v1beta1/hyperband/service.py (SURVEY.md §8(a) A10) [RECALL].

Integer bracket bookkeeping (Li et al., "Hyperband", JMLR 2018, Alg. 1): s_max = ⌊log_η r_l⌋, and for bracket s
n = ⌈(s_max+1)/(s+1)·η^s⌉ configurations start at resource r = r_l·η^{-s}; rung i keeps the best ⌊n_i/η⌋ and multiplies
the resource by η.  The state round-trips through ``reply.algorithm.algorithm_settings`` (the service is stateless, as
upstream's is): ``current_s``, ``current_i``, ``n``, ``r``, ``evaluating_trials``, plus ``bracket_trials`` — the names of
the trials of the rung being evaluated.  This is host-side logic by nature (tens of integers and one top-k over at most a
few thousand finished trials per call); there is nothing for the GPU to do here and none is used.
"""
from __future__ import annotations

import math
import threading

import numpy as np

from . import api_pb as api
from .internal import MAX_GOAL, AlgorithmSettingsError, HyperParameterSearchSpace, Trial, parse_settings
from .service import _Base, _reply_from


def bracket_plan(eta: float, r_l: float):
    """[(s, n, r)] for s = s_max .. 0 — the table the tests check against the paper's formula."""
    s_max = int(math.floor(math.log(r_l) / math.log(eta) + 1e-9))
    return [(s, int(math.ceil((s_max + 1) / (s + 1) * eta ** s)), r_l * eta ** (-s)) for s in range(s_max, -1, -1)]


class HyperBandParam:
    def __init__(self, settings: dict):
        try:
            self.eta = float(settings.get("eta", 3))
            self.r_l = float(settings["r_l"])
        except KeyError:
            raise AlgorithmSettingsError("r_l must be set for hyperband")
        except ValueError:
            raise AlgorithmSettingsError("eta and r_l must be numbers")
        if self.eta <= 1:
            raise AlgorithmSettingsError(f"eta should be greater than 1, got {self.eta}")
        if self.r_l <= 0:
            raise AlgorithmSettingsError(f"r_l should be positive, got {self.r_l}")
        self.resource_name = settings.get("resource_name", "")
        if not self.resource_name:
            raise AlgorithmSettingsError("resource_name must be set for hyperband")
        self.s_max = int(math.floor(math.log(self.r_l) / math.log(self.eta) + 1e-9))
        self.b_l = (self.s_max + 1) * self.r_l
        self.current_s = int(settings.get("current_s", self.s_max))
        self.current_i = int(settings.get("current_i", 0))
        self.n = int(settings.get("n", -1))
        self.r = float(settings.get("r", -1))
        self.evaluating_trials = int(settings.get("evaluating_trials", 0))
        self.bracket_trials = [t for t in settings.get("bracket_trials", "").split(",") if t]
        self.random_state = int(settings["random_state"]) if "random_state" in settings else None

    def start_bracket(self, s):
        self.current_s, self.current_i = s, 0
        self.n = int(math.ceil((self.s_max + 1) / (s + 1) * self.eta ** s))
        self.r = self.r_l * self.eta ** (-s)

    def to_settings(self):
        return {"eta": repr(self.eta), "r_l": repr(self.r_l), "resource_name": self.resource_name, "current_s": str(self.current_s),
                "current_i": str(self.current_i), "n": str(self.n), "r": repr(self.r), "evaluating_trials": str(self.evaluating_trials),
                "bracket_trials": ",".join(self.bracket_trials),
                **({"random_state": str(self.random_state)} if self.random_state is not None else {})}


class HyperbandService(_Base):
    algorithm_names = ("hyperband",)

    def __init__(self):
        self._lock = threading.Lock()
        self._calls = {}

    def validate(self, experiment):
        self.check_algorithm(experiment)
        ss = HyperParameterSearchSpace.convert(experiment)
        p = HyperBandParam(parse_settings(experiment))
        if p.resource_name not in [q.name for q in ss.params]:
            raise AlgorithmSettingsError(f"resource_name {p.resource_name} is not in the search space")

    @staticmethod
    def _resource_value(param_spec, r):
        return str(int(round(r))) if param_spec.type == "int" else repr(float(r))

    def get_suggestions(self, request):
        from .internal import Assignment
        exp = request.experiment
        ss = HyperParameterSearchSpace.convert(exp)
        p = HyperBandParam(parse_settings(exp))
        res_spec = next((q for q in ss.params if q.name == p.resource_name), None)
        if res_spec is None:
            raise AlgorithmSettingsError(f"resource_name {p.resource_name} is not in the search space")
        trials = {t.name: t for t in Trial.convert(request.trials)}
        lists = []
        if p.evaluating_trials == 0 and not p.bracket_trials:                       # first call: master bracket s_max
            if p.n < 0:
                p.start_bracket(p.s_max)
            lists = self._master(ss, p, res_spec, exp.name)
        else:
            if p.bracket_trials:
                done = [trials[n] for n in p.bracket_trials if n in trials]
                expected = len(p.bracket_trials)
            else:   # a controller that only echoes the counters (upstream's behaviour): the rung = the most recent finished trials
                done = list(trials.values())[-p.evaluating_trials:] if p.evaluating_trials else []
                expected = p.evaluating_trials
            if len(done) < expected:
                # the rung is still running: nothing new to hand out (Katib re-asks later)
                return self._reply(lists, p)
            sign = -1.0 if ss.goal == MAX_GOAL else 1.0
            order = np.argsort([sign * float(t.target_metric.value) for t in done], kind="stable")
            n_i = len(done)
            keep = int(math.floor(n_i / p.eta))
            if p.current_i < p.current_s and keep >= 1:                                 # child rung: top n_i/η, η× the resource
                p.current_i += 1
                r_i = p.r * p.eta ** p.current_i
                for k in order[:keep]:
                    t = done[int(k)]
                    lists.append([Assignment(a.name, self._resource_value(res_spec, r_i) if a.name == p.resource_name else a.value)
                                  for a in t.assignments])
            else:                                                                       # bracket finished → next s (or wrap around)
                p.start_bracket(p.current_s - 1 if p.current_s > 0 else p.s_max)
                lists = self._master(ss, p, res_spec, exp.name)
        p.evaluating_trials = len(lists)
        # names are assigned by the controller after this reply: it must echo them back in `bracket_trials` (upstream keeps a
        # count only); when it does not, fall back to "the last evaluating_trials finished trials"
        p.bracket_trials = []
        return self._reply(lists, p)

    def _master(self, ss, p, res_spec, exp_name):
        from ..space import Space
        from .base_service import BaseSkoptService, dimensions
        with self._lock:
            k = self._calls.get(exp_name, 0)
            self._calls[exp_name] = k + 1
        rng = np.random.default_rng(None if p.random_state is None else [p.random_state, p.current_s, k])
        space = Space(dimensions(ss))
        pts = space.inverse_transform(space.rvs_transformed(p.n, rng, np.float64))
        out = []
        for pt in pts:
            a = BaseSkoptService.convert(ss, pt)
            for x in a:
                if x.name == p.resource_name:
                    x.value = self._resource_value(res_spec, p.r)
            out.append(a)
        return out

    @staticmethod
    def _reply(lists, p):
        reply = _reply_from(lists)
        reply.algorithm.algorithm_name = "hyperband"
        for k, v in p.to_settings().items():
            s = reply.algorithm.algorithm_settings.add()
            s.name, s.value = k, v
        return reply
