"""``api.v1.beta1.Suggestion`` servicers.

* ``SkoptService``  — algorithm ``bayesianoptimization`` (kubeflow/katib pkg/suggestion/v1beta1/skopt/service.py):
  GetSuggestions → BaseSkoptService → kubeflow_b200.Optimizer → libkbo (GPU), with base_estimator GP, RF or ET (GBRT is
  refused).  ValidateAlgorithmSettings accepts the upstream settings (base_estimator, n_initial_points, acq_func,
  acq_optimizer, random_state) plus engine knobs as EXTRA settings, so an unchanged Experiment works and an extended one
  can opt in (SURVEY.md §5 "config"); the GP-only knobs are refused with a tree estimator.
* ``RandomService`` — algorithm ``random`` (upstream: the hyperopt service's random search): BASELINE.json config 1,
  gRPC plumbing on CPU, no GPU involved.
Errors: bad settings → INVALID_ARGUMENT; anything else → INTERNAL (SURVEY.md §8(b)).
"""
from __future__ import annotations

import logging
import threading

import grpc
import numpy as np

from . import api_pb as api
from .internal import (AlgorithmSettingsError, HyperParameterSearchSpace, Trial, parse_settings)

logger = logging.getLogger(__name__)

SKOPT_SETTINGS = ("base_estimator", "n_initial_points", "acq_func", "acq_optimizer", "random_state")
ENGINE_SETTINGS = {"n_points": int, "kernel": str, "length_scale": float, "amplitude": float, "noise": float, "xi": float,
                   "kappa": float, "var_mode": str, "theta_grid": int, "theta_search": int, "theta_fit": str, "theta_fit_maxiter": int, "theta_restarts": int, "ard": int, "device": int,
                   "candidate_backend": str}

TREE_ESTIMATORS = {"RF": "RandomForestRegressor", "ET": "ExtraTreesRegressor"}   # skopt's cook_estimator names
GP_ONLY_SETTINGS = ("kernel", "length_scale", "amplitude", "noise", "var_mode", "theta_grid", "theta_search", "theta_fit",
                    "theta_fit_maxiter", "theta_restarts", "ard")
# what theta_fit: skopt takes from skopt itself (its start, its bounds, its search): an Experiment may not set them beside it
SKOPT_THETA_EXCLUSIVE = ("theta_grid", "theta_search", "ard", "length_scale", "amplitude", "noise")


def validate_skopt_settings(settings: dict) -> dict:
    """Returns the parsed keyword arguments or raises AlgorithmSettingsError (mirrors upstream OptimizerConfiguration)."""
    out = {}
    for name, value in settings.items():
        try:
            if name == "base_estimator":
                if value not in ("GP", "RF", "ET", "GBRT"):
                    raise AlgorithmSettingsError(f"base_estimator {value} is not supported in Bayesian optimization")
                if value == "GBRT":
                    raise AlgorithmSettingsError(f"base_estimator {value}: only GP runs on the GPU engine")
                out[name] = value
            elif name == "n_initial_points":
                if int(value) < 0:
                    raise AlgorithmSettingsError(f"n_initial_points should be great or equal than zero, got {value}")
                out[name] = int(value)
            elif name == "acq_func":
                if value not in ("gp_hedge", "LCB", "EI", "PI", "EIps", "PIps"):
                    raise AlgorithmSettingsError(f"acq_func {value} is not supported in Bayesian optimization")
                out[name] = value
            elif name == "acq_optimizer":
                if value not in ("auto", "sampling", "lbfgs"):
                    raise AlgorithmSettingsError(f"acq_optimizer {value} is not supported in Bayesian optimization")
                out[name] = value
            elif name == "random_state":
                if int(value) < 0:
                    raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {value}")
                out[name] = int(value)
            elif name in ENGINE_SETTINGS:
                v = ENGINE_SETTINGS[name](value)
                if name == "kernel" and v not in ("rbf", "matern52", "hamming"):
                    raise AlgorithmSettingsError(f"kernel {v} must be rbf, matern52 or hamming")
                if name == "var_mode" and v not in ("tc", "f64", "auto"):
                    raise AlgorithmSettingsError(f"var_mode {v} must be tc, f64 or auto")
                if name == "candidate_backend" and v not in ("torch", "numpy"):
                    raise AlgorithmSettingsError(f"candidate_backend {v} must be torch or numpy")
                if name == "theta_fit" and v not in ("lbfgs", "skopt"):
                    raise AlgorithmSettingsError(f"theta_fit {v} must be lbfgs or skopt")
                if name in ("theta_search", "theta_restarts") and v < 0:
                    raise AlgorithmSettingsError(f"{name} must be >= 0, got {value}")
                if name in ("n_points", "theta_grid") and v < 1:
                    raise AlgorithmSettingsError(f"{name} must be >= 1, got {value}")
                if name in ("length_scale", "amplitude") and not v > 0:
                    raise AlgorithmSettingsError(f"{name} must be > 0, got {value}")
                if name == "noise" and v < 0:
                    raise AlgorithmSettingsError(f"noise must be >= 0, got {value}")
                out[name] = v
            else:
                raise AlgorithmSettingsError(f"unknown setting {name} for algorithm bayesianoptimization")
        except AlgorithmSettingsError:
            raise
        except (TypeError, ValueError):
            raise AlgorithmSettingsError(f"failed to convert {value!r} for setting {name}")
    if out.get("base_estimator") in TREE_ESTIMATORS:
        est = out["base_estimator"]
        if out.get("acq_optimizer") == "lbfgs":      # skopt's Optimizer refuses it: trees have no gradients
            raise AlgorithmSettingsError(f"The regressor {TREE_ESTIMATORS[est]} should run with acq_optimizer='sampling'.")
        for name in GP_ONLY_SETTINGS:
            if name in out:
                raise AlgorithmSettingsError(f"setting {name} applies to base_estimator GP only, not {est}")
    if out.get("theta_fit") == "skopt":
        for name in SKOPT_THETA_EXCLUSIVE:
            if name in out and not (name == "theta_grid" and out[name] == 1) and not (name in ("theta_search", "ard") and out[name] == 0):
                raise AlgorithmSettingsError(f"setting {name} cannot be combined with theta_fit skopt, which uses skopt's own start and bounds")
    elif "theta_restarts" in out:
        raise AlgorithmSettingsError("setting theta_restarts applies to theta_fit skopt only")
    if out.get("kernel") == "hamming":   # these search the one-hot columns' length scales, which Hamming weights replace
        for name, given in (("theta_grid", out.get("theta_grid", 1) > 1), ("theta_search", out.get("theta_search", 0) > 0),
                            ("theta_fit", out.get("theta_fit") == "lbfgs")):
            if given:
                raise AlgorithmSettingsError(f"setting {name} {out[name]} cannot be combined with kernel hamming")
    return out


def check_kernel_space(settings: dict, search_space):
    """skopt's HammingKernel is its model of all-categorical spaces only: ``kernel: hamming`` beside a ``double`` or ``int``
    parameter is refused, naming it."""
    if settings.get("kernel") != "hamming":
        return
    from .internal import CATEGORICAL, DISCRETE
    for p in search_space.params:
        if p.type not in (CATEGORICAL, DISCRETE):
            raise AlgorithmSettingsError(f"kernel hamming needs every parameter categorical or discrete: parameter {p.name} is {p.type}")


def experiment_fingerprint(exp, search_space, settings: dict) -> tuple:
    """What a cached per-experiment state depends on: goal, objective metric, the search space and the parsed settings."""
    return (search_space.goal, exp.spec.objective.objective_metric_name,
            tuple((p.name, p.type, p.min, p.max, tuple(p.list), p.step) for p in search_space.params),
            tuple(sorted((k, repr(v)) for k, v in settings.items())))


def _reply_from(assignment_lists) -> "api.GetSuggestionsReply":
    reply = api.GetSuggestionsReply()
    for assignments in assignment_lists:
        pa = reply.parameter_assignments.add()
        for a in assignments:
            x = pa.assignments.add()
            x.name, x.value = a.name, a.value
    return reply


class _Base:
    """A servicer for ``algorithm_names``.  The services that keep per-experiment state hold it in ``_exps`` (experiment name ->
    entry with ``close()``, least recently used first), reached through ``experiment()`` under ``_lock``; ``engine_defaults``
    are settings (``device``, ...) an Experiment may override."""
    algorithm_names: tuple = ()
    MAX_EXPERIMENTS = 8           # entries own libkbo handles (device memory): bound how many live at once

    def __init__(self, engine_defaults: dict | None = None, max_experiments: int | None = None):
        self._lock = threading.Lock()       # handlers may run concurrently (grpc thread pool): GPU work is serialised here
        self._exps = {}
        self.engine_defaults = dict(engine_defaults or {})
        self.max_experiments = int(self.MAX_EXPERIMENTS if max_experiments is None else max_experiments)

    def check_algorithm(self, experiment, allow_empty: bool = False):
        name = experiment.spec.algorithm.algorithm_name
        if name not in self.algorithm_names and not (allow_empty and name == ""):
            raise AlgorithmSettingsError(f"unknown algorithm name {name}")

    def with_defaults(self, raw: dict, settings: dict) -> dict:
        """``settings`` (parsed from the Experiment's ``raw`` settings) plus the engine defaults it does not set."""
        return {**settings, **{k: v for k, v in self.engine_defaults.items() if k not in raw}}

    def experiment(self, name: str, fingerprint, make):
        """The per-experiment state of ``name``, made by ``make()`` when absent.  An experiment recreated under the same name,
        or whose search space / objective / settings changed, must not meet the old state (old dimensions, old history, old
        settings): an entry is valid for one fingerprint only, and a stale one is closed and replaced.  Past
        ``max_experiments`` the least recently used entries are closed and dropped.  Call with ``_lock`` held."""
        entry = self._exps.get(name)
        if entry is not None and entry.fingerprint != fingerprint:
            self._exps.pop(name).close()
            entry = None
        if entry is None:
            entry = make()
            entry.fingerprint = fingerprint
            self._exps[name] = entry
            while len(self._exps) > self.max_experiments:
                self._exps.pop(next(iter(self._exps))).close()
        else:
            self._exps[name] = self._exps.pop(name)      # mark as most recently used
        return entry

    def _abort(self, context, code, msg):
        logger.warning("%s: %s", code, msg)
        context.set_code(code)
        context.set_details(msg)

    def ValidateAlgorithmSettings(self, request, context):
        try:
            self.validate(request.experiment)
        except AlgorithmSettingsError as e:
            self._abort(context, grpc.StatusCode.INVALID_ARGUMENT, str(e))
        except Exception as e:  # noqa: BLE001
            self._abort(context, grpc.StatusCode.INTERNAL, f"{type(e).__name__}: {e}")
        return api.ValidateAlgorithmSettingsReply()

    def GetSuggestions(self, request, context):
        try:
            return self.get_suggestions(request)
        except (AlgorithmSettingsError,) as e:
            self._abort(context, grpc.StatusCode.INVALID_ARGUMENT, str(e))
        except ValueError as e:
            self._abort(context, grpc.StatusCode.INVALID_ARGUMENT, str(e))
        except Exception as e:  # noqa: BLE001  (CUDA errors, not-PD, ...)
            logger.exception("GetSuggestions failed")
            self._abort(context, grpc.StatusCode.INTERNAL, f"{type(e).__name__}: {e}")
        return api.GetSuggestionsReply()


class SkoptService(_Base):
    algorithm_names = ("bayesianoptimization",)

    def __init__(self, engine_defaults: dict | None = None, max_experiments: int | None = None):
        super().__init__(engine_defaults, max_experiments)
        self.last_ingest = None             # "scan" | "messages": how the last request's trials reached the optimizer

    @property
    def _services(self) -> dict:
        """experiment name -> BaseSkoptService (the per-experiment cache under the name the benchmark and tests read)."""
        return self._exps

    def validate(self, experiment):
        self.check_algorithm(experiment)
        search_space = HyperParameterSearchSpace.convert(experiment)
        check_kernel_space(validate_skopt_settings(parse_settings(experiment)), search_space)

    def get_suggestions(self, request):
        from .base_service import BaseSkoptService
        from .ingest import LazyRequest
        exp = request.experiment
        self.check_algorithm(exp, allow_empty=True)
        search_space = HyperParameterSearchSpace.convert(exp)
        raw = parse_settings(exp)
        settings = validate_skopt_settings(raw)
        check_kernel_space(settings, search_space)
        lazy = request if isinstance(request, LazyRequest) and request.scanned else None
        fingerprint = experiment_fingerprint(exp, search_space, settings)
        with self._lock:
            svc = self.experiment(exp.name, fingerprint,
                                  lambda: BaseSkoptService(search_space=search_space, **self.with_defaults(raw, settings)))
            # the wire scan tells the new trials from flat arrays; it declines (False) whenever a trial needs the message walk
            self.last_ingest = "scan" if (lazy is not None and svc.ingest(lazy)) else "messages"
            trials = [] if self.last_ingest == "scan" else Trial.convert(request.trials, skip_names=svc.told_trials)
            lists = svc.getSuggestions(trials, max(int(request.current_request_number), 0))
        return _reply_from(lists)


def prior_points(ss, rng, n: int) -> list:
    """n uniform random points of the search space (integers uniform over [min, max], categories uniform), in parameter
    values — the sampling of Katib's ``random`` algorithm, shared with ``tpe``'s start-up phase."""
    from ..space import Space
    from .base_service import dimensions
    space = Space(dimensions(ss))
    return space.inverse_transform(space.rvs_transformed(n, rng, np.float64)) if n else []


class RandomService(_Base):
    """Uniform random search over the feasible space (Katib algorithm ``random``); CPU only."""
    algorithm_names = ("random",)

    def __init__(self):
        self._rngs = {}
        self._lock = threading.Lock()

    def validate(self, experiment):
        self.check_algorithm(experiment)
        HyperParameterSearchSpace.convert(experiment)
        for k, v in parse_settings(experiment).items():
            if k != "random_state":
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm random")
            try:
                if int(v) < 0:
                    raise ValueError
            except ValueError:
                raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")

    def get_suggestions(self, request):
        from .base_service import BaseSkoptService
        exp = request.experiment
        ss = HyperParameterSearchSpace.convert(exp)
        st = parse_settings(exp)
        with self._lock:
            rng = self._rngs.get(exp.name)
            if rng is None:
                rng = self._rngs[exp.name] = np.random.default_rng(int(st["random_state"]) if "random_state" in st else None)
            pts = prior_points(ss, rng, max(int(request.current_request_number), 0))
        return _reply_from([BaseSkoptService.convert(ss, p) for p in pts])


class SobolService(_Base):
    """Quasi-random search over the feasible space (Katib algorithm ``sobol``, the second sampler of the goptuna service;
    SURVEY.md §2 row 18).  Scrambled Sobol points from SciPy's QMC engine, mapped through the same space transform as every
    other algorithm here; stateless across calls by skipping the points already handed out (= number of trials seen +
    number requested so far).  CPU only — there is no arithmetic to accelerate."""
    algorithm_names = ("sobol",)

    def __init__(self):
        self._lock = threading.Lock()
        self._issued = {}

    def validate(self, experiment):
        self.check_algorithm(experiment)
        ss = HyperParameterSearchSpace.convert(experiment)
        for p in ss.params:
            if p.type in ("categorical", "discrete") and len(p.list) < 1:
                raise AlgorithmSettingsError(f"parameter {p.name!r}: empty feasible list")
        for k, v in parse_settings(experiment).items():
            if k != "random_state":
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm sobol")
            try:
                if int(v) < 0:
                    raise ValueError
            except ValueError:
                raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")

    def get_suggestions(self, request):
        from scipy.stats import qmc
        from ..space import Categorical, Integer
        from .base_service import BaseSkoptService, dimensions
        exp = request.experiment
        ss = HyperParameterSearchSpace.convert(exp)
        st = parse_settings(exp)
        n = max(int(request.current_request_number), 0)
        with self._lock:
            start = self._issued.get(exp.name, 0)
            self._issued[exp.name] = start + n
        if n == 0:
            return _reply_from([])
        eng = qmc.Sobol(d=len(ss.params), scramble=True, seed=int(st.get("random_state", 0)))
        if start:
            eng.fast_forward(start)
        U = eng.random(n)
        dims = dimensions(ss)
        pts = []
        for u in U:
            pt = []
            for d, v in zip(dims, u):
                if isinstance(d, Categorical):
                    pt.append(d.categories[min(int(v * len(d.categories)), len(d.categories) - 1)])
                elif isinstance(d, Integer):
                    pt.append(min(d.low + int(v * (d.high - d.low + 1)), d.high))
                else:
                    pt.append(d.low + float(v) * (d.high - d.low))
            pts.append(pt)
        return _reply_from([BaseSkoptService.convert(ss, p) for p in pts])


class DispatchService(_Base):
    """One endpoint for several algorithms (upstream runs one Deployment per algorithm image; this routes by name)."""

    def __init__(self, services):
        self._by_name = {n: s for s in services for n in s.algorithm_names}

    def _pick(self, experiment):
        name = experiment.spec.algorithm.algorithm_name
        if name not in self._by_name:
            raise AlgorithmSettingsError(f"unknown algorithm name {name!r}; served: {sorted(self._by_name)}")
        return self._by_name[name]

    def validate(self, experiment):
        self._pick(experiment).validate(experiment)

    def get_suggestions(self, request):
        return self._pick(request.experiment).get_suggestions(request)
