"""``cmaes`` — Katib's goptuna-backed CMA-ES algorithm (SURVEY.md §8(a) A9) on the GPU sampler ``kubeflow_b200.cmaes``.

Search happens in the normalised cube [0,1]^D (reals and integers; categorical/discrete parameters are rejected, as
goptuna's CMA sampler does), mean0 = 0.5, sigma0 = 1/6 unless ``sigma`` is set; samples are clipped to the cube.
A generation's λ points are handed out across GetSuggestions calls; when all λ results are back the population is told
and the next generation is sampled.  Samples are tracked BY INDEX: two samples that round or clip to the same assignment
strings (integer parameters, cube boundary) are two pending entries under one key, matched first-in first-out; a sample
whose trial ended without an objective (FAILED / KILLED / METRICSUNAVAILABLE) goes back to the head of the queue and is
handed out again — goptuna likewise keeps sampling the running generation until popsize trials are COMPLETE — so neither
duplicates nor failures can stall the generation.  If the controller asks for more points than the generation has left,
the extra points are independent draws from the current distribution (they do not enter the update), which is what
goptuna's relative/independent sampling split amounts to.  With ``restart_strategy`` ``ipop`` or ``bipop`` the
termination test the sampler runs on the device after every tell is read after each complete generation; when any of
its criteria holds, the run restarts in place on the schedule of ``cma_restart.py`` (IPOP: doubled population; BIPOP:
interlaced large and small runs) with a fresh mean drawn in the cube.  Outstanding samples of the stopped run stay
unmatched, like extra independent draws.  With ``with_margin: true`` the sampler runs CMA-ES with Margin (Optuna's
``CmaEsSampler(with_margin=True)``): ``int`` and numeric ``discrete`` parameters become discrete dimensions whose levels
(``cma_margin.py``) the sampler encodes on the device, and the margin α (``margin``, default 1/(D·λ)) keeps a
coordinate from freezing on one level once σ is small.  Trials get the encoded level's value; a restart resets the margin.
With ``lr_adapt: true`` the sampler runs CMA-ES with learning-rate adaptation (Optuna's ``CmaEsSampler(lr_adapt=True)``,
``oracle/cma_lra_oracle.py``): at the default population it lowers the learning rates of the mean and the covariance
when the signal-to-noise ratio of their updates falls, as on a noisy or multimodal objective, instead of asking for a
larger ``popsize``.  It works with ``popsize``, ``sigma`` and ``restart_strategy`` (each restart starts the adaptation
afresh) and is refused beside ``with_margin: true``.
With ``use_separable_cma: true`` the sampler runs separable CMA-ES (Optuna's ``CmaEsSampler(use_separable_cma=True)``,
``oracle/sepcma_oracle.py``): C is kept as its diagonal, so a generation costs O(λ·D) and spaces of up to 4096 parameters
are served (the full sampler stops at 128); per-coordinate scales are learnt faster, correlations between parameters are
not learnt at all.  It works with ``popsize``, ``sigma``, ``random_state`` and ``restart_strategy`` and is refused beside
``with_margin: true`` and beside ``lr_adapt: true``, as Optuna refuses both.

Each experiment's sampler is kept for one fingerprint of its search space, objective and settings: an experiment recreated
under the same name with a changed space or changed settings starts a new run, and the old sampler is closed.  At most
``max_experiments`` (default 64) samplers live at once; past that the least recently used is closed.  A CMA-ES run is the
sampler's device state and cannot be rebuilt from the trials Katib resends, so an evicted experiment that comes back starts
a new run from the initial mean and σ.
"""
from __future__ import annotations

import numpy as np

from . import api_pb as api
from .internal import (CATEGORICAL, DISCRETE, DOUBLE, INTEGER, MAX_GOAL, AlgorithmSettingsError, Assignment,
                       HyperParameterSearchSpace, Trial, parse_settings)
from .cma_margin import discrete_dims, encode, parse_with_margin
from .cma_restart import STRATEGIES, Schedule
from .service import _Base, _reply_from, experiment_fingerprint

SEP_MAX_PARAMS = 4096          # kbo_sepcma_create's limit


def validate_cmaes_settings(settings: dict, n_params: int) -> dict:
    out = {}
    for k, v in settings.items():
        try:
            if k == "random_state":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")
            elif k == "sigma":
                out[k] = float(v)
                if not out[k] > 0:
                    raise AlgorithmSettingsError(f"sigma should be positive, got {v}")
            elif k == "popsize":
                out[k] = int(v)
                if not 4 <= out[k] <= 8192:
                    raise AlgorithmSettingsError(f"popsize must be in [4, 8192], got {v}")
            elif k in ("restart_strategy", "device"):
                out[k] = v
            elif k in ("with_margin", "lr_adapt", "use_separable_cma"):
                out[k] = parse_with_margin(v, k)
            elif k == "margin":
                out[k] = float(v)
                if not 0.0 < out[k] < 1.0:
                    raise AlgorithmSettingsError(f"margin must be in (0, 1), got {v}")
            else:
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm cmaes")
        except ValueError:
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
    if "margin" in out and not out.get("with_margin", False):
        raise AlgorithmSettingsError("margin needs with_margin: true")
    if out.get("lr_adapt", False) and out.get("with_margin", False):
        raise AlgorithmSettingsError("lr_adapt: true cannot be combined with with_margin: true")
    if out.get("use_separable_cma", False):
        for other in ("with_margin", "lr_adapt"):
            if out.get(other, False):
                raise AlgorithmSettingsError(f"use_separable_cma: true cannot be combined with {other}: true")
        if n_params > SEP_MAX_PARAMS:
            raise AlgorithmSettingsError(f"use_separable_cma supports at most {SEP_MAX_PARAMS} parameters, got {n_params}")
    if out.get("restart_strategy", "none") not in STRATEGIES:
        raise AlgorithmSettingsError(f"restart_strategy must be one of {', '.join(STRATEGIES)}, got {out['restart_strategy']!r}")
    if n_params < 2:
        raise AlgorithmSettingsError("cmaes only supports two or more dimensional continuous search space")   # goptuna's rule
    return out


class _Experiment:
    def __init__(self, space, D, settings):
        from .. import cmaes
        self.sep = settings.get("use_separable_cma", False)
        self.es = (cmaes.SepCmaEs if self.sep else cmaes.CmaEs)(np.full(D, 0.5), settings.get("sigma", 1.0 / 6.0), popsize=settings.get("popsize"),
                        seed=settings.get("random_state", 0), device=int(settings.get("device", 0)))
        self.queue = []          # [(sample index, assignments)] of the current generation not handed out yet
        self.assign = {}         # sample index -> assignments of the current generation
        self.pending = {}        # key -> [sample indices handed out, no result yet] (first in, first out)
        self.fitness = {}        # sample index -> value
        self.seen = set()        # trial names already accounted for (finished with or without an objective)
        self.extra_rng = np.random.default_rng(settings.get("random_state", 0) + 7919)
        strategy = settings.get("restart_strategy", "none")
        # IPOP / BIPOP: λ0, σ0, the restart draws and the BIPOP budgets live in the schedule; None = one run, no test read
        self.schedule = None if strategy == "none" else Schedule(strategy, D, settings.get("popsize"), settings.get("sigma", 1.0 / 6.0),
                                                                   settings.get("random_state", 0))
        self.run_gens = 0        # generations told in the current run
        # with_margin: {parameter index: Levels} of the discrete dimensions, encoded by the sampler
        self.levels = discrete_dims(space.params) if settings.get("with_margin", False) else {}
        if self.levels:
            self.es.set_margin({j: L.cube for j, L in self.levels.items()}, settings.get("margin"))
        if settings.get("lr_adapt", False):
            self.es.set_lr_adapt(True)

    def close(self):
        self.es.close()


class CmaesService(_Base):
    algorithm_names = ("cmaes",)
    MAX_EXPERIMENTS = 64          # an evicted run cannot be rebuilt from the trials (module docstring)

    @staticmethod
    def _space(experiment):
        ss = HyperParameterSearchSpace.convert(experiment)
        margin = any(s.name == "with_margin" and str(s.value).strip().lower() == "true"
                     for s in experiment.spec.algorithm.algorithm_settings)
        for p in ss.params:
            if p.type == CATEGORICAL or (p.type == DISCRETE and not margin):
                raise AlgorithmSettingsError(f"cmaes does not support categorical/discrete parameter {p.name!r}")
        return ss

    def validate(self, experiment):
        self.check_algorithm(experiment)
        ss = self._space(experiment)
        if validate_cmaes_settings(parse_settings(experiment), len(ss.params)).get("with_margin", False):
            discrete_dims(ss.params)

    @staticmethod
    def _to_assignments(ss, u, levels=None):
        out = []
        for j, (p, v) in enumerate(zip(ss.params, np.clip(u, 0.0, 1.0))):
            if levels and j in levels:
                out.append(Assignment(p.name, levels[j].value(float(u[j]))))
                continue
            lo, hi = float(p.min), float(p.max)
            x = lo + float(v) * (hi - lo)
            out.append(Assignment(p.name, str(int(round(x))) if p.type == INTEGER else repr(x)))
        return out

    @staticmethod
    def _key(assignments):
        return tuple((a.name, a.value) for a in assignments)

    def _new_generation(self, st, ss):
        X = st.es.ask().cpu().numpy()
        st.queue = [(i, self._to_assignments(ss, X[i], st.levels)) for i in range(X.shape[0])]
        st.assign = {i: a for i, a in st.queue}
        st.pending = {}
        st.fitness = {}

    def get_suggestions(self, request):
        exp = request.experiment
        ss = self._space(exp)
        raw = parse_settings(exp)
        settings = self.with_defaults(raw, validate_cmaes_settings(raw, len(ss.params)))
        trials = Trial.convert(request.trials)
        sign = -1.0 if ss.goal == MAX_GOAL else 1.0
        with self._lock:
            def make():
                st = _Experiment(ss, len(ss.params), settings)
                self._new_generation(st, ss)
                return st
            st = self.experiment(exp.name, experiment_fingerprint(exp, ss, settings), make)
            for t in trials:
                if t.name in st.seen:
                    continue
                st.seen.add(t.name)
                waiting = st.pending.get(self._key(t.assignments))
                if waiting:
                    st.fitness[waiting.pop(0)] = sign * float(t.target_metric.value)
            # trials that ended without an objective: their sample is handed out again
            for t in request.trials:
                # (a SUCCEEDED / EARLYSTOPPED trial still unseen here carried no objective metric: same treatment)
                if t.name in st.seen or t.status.condition not in (api.FAILED, api.KILLED, api.METRICSUNAVAILABLE, api.SUCCEEDED,
                                                                   api.EARLYSTOPPED):
                    continue
                st.seen.add(t.name)
                waiting = st.pending.get(self._key(Assignment.convert(t.spec.parameter_assignments.assignments)))
                if waiting:
                    i = waiting.pop(0)
                    st.queue.insert(0, (i, st.assign[i]))
            if len(st.fitness) == st.es.popsize:
                st.es.tell(np.array([st.fitness[i] for i in range(st.es.popsize)]))
                st.run_gens += 1
                if st.schedule is not None and st.es.stop_flags()[0]:
                    lam, mean, sigma = st.schedule.next_run(st.es.popsize, st.run_gens)
                    st.es.restart(lam, mean, sigma)
                    st.run_gens = 0
                self._new_generation(st, ss)
            lists = []
            for _ in range(max(int(request.current_request_number), 0)):
                if st.queue:
                    i, a = st.queue.pop(0)
                    st.pending.setdefault(self._key(a), []).append(i)
                    lists.append(a)
                else:   # generation exhausted but not finished: independent draw from the current distribution
                    s = st.es.state()
                    z = st.extra_rng.standard_normal(st.es.D)
                    if st.levels:
                        x = s["mean"] + s["sigma"] * (st.es.margin_state()["A"] * (s["B"] @ (s["d"] * z)))
                        lists.append(self._to_assignments(ss, encode(st.levels, x), st.levels))
                    elif st.sep:
                        lists.append(self._to_assignments(ss, s["mean"] + s["sigma"] * (s["d"] * z)))
                    else:
                        lists.append(self._to_assignments(ss, s["mean"] + s["sigma"] * (s["B"] @ (s["d"] * z))))
        return _reply_from(lists)
