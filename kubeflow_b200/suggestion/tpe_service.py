"""``tpe`` — Katib's hyperopt-backed Tree-structured Parzen Estimator (the second algorithm of the upstream hyperopt image) on
the GPU engine ``kubeflow_b200.tpe`` (contract: oracle/tpe_oracle.py).

* Space: DOUBLE → uniform(min, max) (``step`` ignored, as the other services here ignore it); INT → quniform(min, max, q), q =
  ``step`` or 1, reported as integers; CATEGORICAL / DISCRETE → choice(list), observed as the category index.
* History: the usable trials (``Trial.convert``), each told once by name, kept in the order first told; loss = objective value,
  negated for MAXIMIZE.
* While fewer than ``n_startup_jobs`` trials are told, points come from the prior — the sampling ``random`` uses — and no GPU
  handle exists.  Then every request scores ``n_EI_candidates`` draws per parameter and point on the device.
* Batches (``current_request_number`` = k > 1): every point gets its own independent draws against the same model, with no
  lies in between.  [RECALL] hyperopt 0.2's ``tpe.suggest`` builds the posterior once per call and draws each new id's
  candidates from it in turn, which is the same thing up to the random stream; Katib's hyperopt service passes
  ``n_startup_jobs = current_request_number`` to it, where this service honours the ``n_startup_jobs`` setting.
* Draws are keyed by (random_state, ask counter, point, parameter, candidate): the same request sequence gives the same
  replies.
* Under the SPMD server (engine default ``shard``, never an Experiment setting) every rank holds the same experiment and
  scores its block of each request's candidates; the replies are those of one GPU.  A seed drawn from fresh entropy is drawn
  on rank 0 and broadcast, and an experiment whose sharded ask failed on any rank is closed on every rank, so the next
  request rebuilds it identically everywhere.
"""
from __future__ import annotations

import numpy as np

from .internal import (DISCRETE, DOUBLE, INTEGER, MAX_GOAL, AlgorithmSettingsError, HyperParameterSearchSpace, Trial,
                       parse_settings, Assignment)
from .service import _Base, _reply_from, experiment_fingerprint, prior_points

MAX_EI_CANDIDATES = 1 << 24


def validate_tpe_settings(settings: dict) -> dict:
    """Parsed settings with defaults, or AlgorithmSettingsError naming the setting [RECALL: Katib's hyperopt validation]."""
    out = dict(gamma=0.25, prior_weight=1.0, n_EI_candidates=24, n_startup_jobs=20)
    for k, v in settings.items():
        try:
            if k == "gamma":
                out[k] = float(v)
                if not 0.0 < out[k] < 1.0:
                    raise AlgorithmSettingsError(f"gamma should be in the range of (0, 1), got {v}")
            elif k == "prior_weight":
                out[k] = float(v)
                if not (out[k] > 0.0 and np.isfinite(out[k])):
                    raise AlgorithmSettingsError(f"prior_weight should be greater than zero, got {v}")
            elif k == "n_EI_candidates":
                out[k] = int(v)
                if not 1 <= out[k] <= MAX_EI_CANDIDATES:
                    raise AlgorithmSettingsError(f"n_EI_candidates should be in [1, 2^24], got {v}")
            elif k == "n_startup_jobs":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"n_startup_jobs should be great or equal than zero, got {v}")
            elif k == "random_state":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")
            elif k == "device":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"device should be great or equal than zero, got {v}")
            else:
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm tpe")
        except AlgorithmSettingsError:
            raise
        except (TypeError, ValueError):
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
    return out


def tpe_space(ss) -> list:
    """The engine's parameter list for a Katib search space."""
    out = []
    for p in ss.params:
        if p.type == DOUBLE:
            out.append(("uniform", float(p.min), float(p.max)))
        elif p.type == INTEGER:
            q = float(p.step) if p.step else 1.0
            if not q > 0:
                raise AlgorithmSettingsError(f"parameter {p.name!r}: step must be > 0, got {p.step}")
            out.append(("quniform", float(p.min), float(p.max), q))
        else:
            out.append(("choice", len(p.list)))
    return out


class _Experiment:
    def __init__(self, ss, settings):
        self.ss, self.settings = ss, settings
        self.space = tpe_space(ss)
        self.rows, self.losses, self.told = [], [], set()
        entropy = settings.get("random_state")
        if entropy is None and settings.get("shard"):      # the ranks' engines must draw the same candidates
            from ..dist import rank0_seed
            entropy = rank0_seed()
        self.rng = np.random.default_rng(entropy)       # start-up phase (None: fresh entropy)
        self.seed = settings["random_state"] if "random_state" in settings else int(self.rng.integers(1 << 62))
        self.engine = None       # kubeflow_b200.tpe.Tpe, created at the first model-based ask
        self.n_engine = 0        # rows told to the engine

    def close(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None

    def row(self, trial) -> list:
        by_name = {a.name: a.value for a in trial.assignments}
        row = []
        for p in self.ss.params:
            v = by_name.get(p.name)
            if v is None:
                raise ValueError(f"trial {trial.name!r} has no assignment for parameter {p.name!r}")
            if p.type in (DOUBLE, INTEGER):
                row.append(float(v))
            elif v in p.list:
                row.append(float(p.list.index(v)))
            else:
                hit = [i for i, c in enumerate(p.list) if p.type == DISCRETE and _same_number(c, v)]
                if not hit:
                    raise ValueError(f"trial {trial.name!r}: {v!r} is not in the feasible list of {p.name!r}")
                row.append(float(hit[0]))
        return row

    def ingest(self, trials, goal, skip_nan: bool = False):
        """Take the request's new usable trials (each name once) into the history, in the order first seen; loss = objective,
        negated for MAXIMIZE.  ``skip_nan``: a NaN objective is marked as seen but never told.  Nothing is taken unless every new
        trial converts: a bad one fails the request."""
        rows, losses, names = [], [], set()
        for t in Trial.convert(trials, skip_names=self.told):
            if t.name in names:
                continue
            names.add(t.name)
            loss = float(t.target_metric.value)
            if skip_nan and np.isnan(loss):
                continue
            rows.append(self.row(t))
            losses.append(-loss if goal == MAX_GOAL else loss)
        self.rows += rows
        self.losses += losses
        self.told.update(names)

    def points(self, k: int, n_startup: int, n_candidates: int, make_engine, shard: bool = False) -> list:
        """k assignment lists: start-up points from the prior (no engine) while fewer than ``n_startup`` trials are told, else
        the engine's (made by ``make_engine()`` on first use), told every trial it has not seen; ``shard``: its sharded ask."""
        if k == 0:
            return []
        if len(self.rows) < n_startup:
            from .base_service import BaseSkoptService
            return [BaseSkoptService.convert(self.ss, p) for p in prior_points(self.ss, self.rng, k)]
        if self.engine is None:
            self.engine = make_engine()
        if self.n_engine < len(self.rows):
            self.engine.tell(np.asarray(self.rows[self.n_engine:]), np.asarray(self.losses[self.n_engine:]))
            self.n_engine = len(self.rows)
        return [self.assignments(x) for x in self.engine.ask(k, n_candidates, shard=shard)]

    def assignments(self, x) -> list:
        out = []
        for p, v in zip(self.ss.params, x):
            if p.type == DOUBLE:
                out.append(Assignment(p.name, repr(float(v))))
            elif p.type == INTEGER:
                out.append(Assignment(p.name, str(int(v))))
            else:
                out.append(Assignment(p.name, str(p.list[int(v)])))
        return out


def _same_number(a: str, b: str) -> bool:
    try:
        return float(a) == float(b)
    except ValueError:
        return False


def sharded_points(service, name: str, st, *args) -> list:
    """``st.points(*args)`` with the service's ``shard`` default; a ``RankFailure`` closes the experiment's entry, which every
    rank does together, so the next request rebuilds it identically everywhere.  Call with ``service._lock`` held."""
    from ..dist import RankFailure
    try:
        return st.points(*args, shard=bool(service.engine_defaults.get("shard")))
    except RankFailure:
        if service._exps.get(name) is st:
            service._exps.pop(name).close()
        raise


class TpeService(_Base):
    algorithm_names = ("tpe",)

    def validate(self, experiment):
        self.check_algorithm(experiment)
        tpe_space(HyperParameterSearchSpace.convert(experiment))
        validate_tpe_settings(parse_settings(experiment))

    def get_suggestions(self, request):
        exp = request.experiment
        self.check_algorithm(exp)
        ss = HyperParameterSearchSpace.convert(exp)
        tpe_space(ss)
        raw = parse_settings(exp)
        settings = self.with_defaults(raw, validate_tpe_settings(raw))
        k = max(int(request.current_request_number), 0)
        with self._lock:
            st = self.experiment(exp.name, experiment_fingerprint(exp, ss, settings), lambda: _Experiment(ss, settings))
            st.ingest(request.trials, ss.goal)

            def make_engine():
                from ..tpe import Tpe
                return Tpe(st.space, gamma=settings["gamma"], prior_weight=settings["prior_weight"], seed=st.seed,
                           device=int(settings.get("device", 0)))
            return _reply_from(sharded_points(self, exp.name, st, k, settings["n_startup_jobs"], settings["n_EI_candidates"], make_engine))
