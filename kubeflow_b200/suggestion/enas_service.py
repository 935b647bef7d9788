"""``enas`` — Katib's neural-architecture search with the ENAS controller on the GPU engine ``kubeflow_b200.enas`` (contract:
oracle/enas_oracle.py, whose docstring lists every recalled detail of the controller; parity with Katib's TF1 service is
unpinned).

* Search space [RECALL: Operation.py]: each ``Operation`` of ``nas_config`` expands into the Cartesian product of its parameter
  specs in spec order, the last spec varying fastest; INT → range(min, max + 1, step), DOUBLE → np.arange(min, max + step, step)
  with an endpoint above max dropped, CATEGORICAL → the list as strings; DISCRETE is refused.  Operation ids number the
  expanded operations 0.. in order.  The experiment has no ``parameter_specs``: HyperParameterSearchSpace is not used.
* Reward [RECALL: service.py]: the mean objective-metric value over the request's SUCCEEDED trials, whatever the objective
  type (EARLYSTOPPED, FAILED and other trials do not count, unlike ``Trial.convert``).
* Calls: the first call of an experiment samples k = ``current_request_number`` arcs without training; every later call with
  at least one SUCCEEDED trial first runs ``controller_train_steps`` REINFORCE steps on the reward; k = 0 replies empty.
  The controller, its Adam moments and its baseline persist across calls in the per-experiment state.
* Reply [RECALL]: per arc, ``architecture`` = json.dumps of the arc organised per layer and ``nn_config`` = json.dumps of
  num_layers, input_sizes, output_sizes and the embedding of the arc's distinct ops in layer order, both with ``"`` replaced
  by ``'``.
* Draws are keyed by (random_state, draw counter, arc, decision): the same request sequence gives the same replies.
"""
from __future__ import annotations

import itertools
import json
import logging

import numpy as np

from . import api_pb as api
from .internal import AlgorithmSettingsError, Assignment, parse_settings, spec_values
from .service import _Base, _reply_from

logger = logging.getLogger(__name__)

NAME = "enas"
MAX_LAYERS, MAX_HIDDEN, MAX_OPS, MAX_REQUEST, MAX_TRAIN_STEPS = 64, 128, 4096, 1024, 10000   # this engine's limits

DEFAULTS = dict(controller_hidden_size=64, controller_temperature=5.0, controller_tanh_const=2.25, controller_entropy_weight=1e-5,
                controller_baseline_decay=0.999, controller_learning_rate=5e-5, controller_skip_target=0.4, controller_skip_weight=0.8,
                controller_train_steps=50, controller_log_every_steps=10)
_NONE_OK = ("controller_temperature", "controller_tanh_const", "controller_entropy_weight", "controller_skip_weight")


def validate_enas_settings(settings: dict) -> dict:
    """Parsed settings with defaults (None where "None" is accepted), or AlgorithmSettingsError naming the setting.  The
    accepted ranges restate upstream's AlgorithmSettings.py from memory [RECALL]; where they are guesses, the oracle says so."""
    out = dict(DEFAULTS)
    for k, v in settings.items():
        try:
            if k in _NONE_OK and str(v) == "None":
                out[k] = None
                continue
            if k in ("controller_hidden_size", "controller_train_steps", "controller_log_every_steps"):
                x = int(v)
                if x < 1:
                    raise AlgorithmSettingsError(f"{k} should be an integer >= 1, got {v}")
                if k == "controller_hidden_size" and x > MAX_HIDDEN:
                    raise AlgorithmSettingsError(f"{k} = {x} exceeds this engine's limit of {MAX_HIDDEN}")
                if k == "controller_train_steps" and x > MAX_TRAIN_STEPS:
                    raise AlgorithmSettingsError(f"{k} = {x} exceeds this engine's limit of {MAX_TRAIN_STEPS}")
            elif k in ("controller_temperature", "controller_tanh_const"):
                x = float(v)
                if not (np.isfinite(x) and x > 0):
                    raise AlgorithmSettingsError(f"{k} should be > 0 or None, got {v}")
            elif k in ("controller_entropy_weight", "controller_skip_weight"):
                x = float(v)
                if not (np.isfinite(x) and x >= 0):
                    raise AlgorithmSettingsError(f"{k} should be >= 0 or None, got {v}")
            elif k == "controller_baseline_decay":
                x = float(v)
                if not 0.0 <= x <= 1.0:
                    raise AlgorithmSettingsError(f"{k} should be in [0, 1], got {v}")
            elif k == "controller_learning_rate":
                x = float(v)
                if not 0.0 < x <= 1.0:
                    raise AlgorithmSettingsError(f"{k} should be in (0, 1], got {v}")
            elif k == "controller_skip_target":
                x = float(v)
                if not 0.0 < x < 1.0:
                    raise AlgorithmSettingsError(f"{k} should be in (0, 1), got {v}")
            elif k in ("random_state", "device"):
                x = int(v)
                if x < 0:
                    raise AlgorithmSettingsError(f"{k} should be greater or equal than zero, got {v}")
            else:
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm {NAME}")
            out[k] = x
        except AlgorithmSettingsError:
            raise
        except (TypeError, ValueError):
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
    return out


def _spec_values(op_type: str, p) -> list:
    where = f"operation {op_type!r}, parameter {p.name!r}"
    if p.parameter_type not in (api.INT, api.DOUBLE, api.CATEGORICAL):
        raise AlgorithmSettingsError(f"{where}: only INT, DOUBLE and CATEGORICAL specs are supported")
    return spec_values(p, where, MAX_OPS)


def expand_operations(operations) -> list:
    """The expanded search space: one dict(opt_id, opt_type, opt_params) per operation id [RECALL: Operation.py]."""
    out = []
    for op in operations:
        if not op.operation_type:
            raise AlgorithmSettingsError("nas_config: every operation needs an operation_type")
        specs = list(op.parameter_specs.parameters)
        if not specs:
            raise AlgorithmSettingsError(f"nas_config: operation {op.operation_type!r} needs at least one parameter spec")
        values = [_spec_values(op.operation_type, p) for p in specs]
        n = int(np.prod([len(v) for v in values], dtype=np.float64))
        if len(out) + n > MAX_OPS:
            raise AlgorithmSettingsError(f"nas_config expands to more than this engine's limit of {MAX_OPS} operations (n_ops)")
        for combo in itertools.product(*values):
            out.append(dict(opt_id=len(out), opt_type=op.operation_type, opt_params={p.name: v for p, v in zip(specs, combo)}))
    if not out:
        raise AlgorithmSettingsError("nas_config needs at least one operation")
    return out


def parse_nas_config(experiment) -> tuple:
    """(num_layers, input_sizes, output_sizes, expanded operations), or AlgorithmSettingsError."""
    nc = experiment.spec.nas_config
    gc = nc.graph_config
    L = int(gc.num_layers)
    if L < 1:
        raise AlgorithmSettingsError(f"nas_config: graph_config.num_layers must be >= 1, got {L}")
    if L > MAX_LAYERS:
        raise AlgorithmSettingsError(f"nas_config: num_layers = {L} exceeds this engine's limit of {MAX_LAYERS}")
    if not len(gc.input_sizes) or not len(gc.output_sizes):
        raise AlgorithmSettingsError("nas_config: graph_config needs non-empty input_sizes and output_sizes")
    return L, [int(x) for x in gc.input_sizes], [int(x) for x in gc.output_sizes], expand_operations(nc.operations.operation)


def organise_arc(arc, L: int) -> list:
    """The flat arc (L(L+1)/2 decisions) per layer: [[op_0], [op_1, skip_0], [op_2, skip_0, skip_1], ...]."""
    arc = [int(x) for x in arc]
    return [arc[l * (l + 1) // 2:(l + 1) * (l + 2) // 2] for l in range(L)]


def nn_config(layers: list, L: int, input_sizes: list, output_sizes: list, ops: list) -> dict:
    emb = {}
    for layer in layers:
        emb.setdefault(layer[0], ops[layer[0]])
    return {"num_layers": L, "input_sizes": input_sizes, "output_sizes": output_sizes, "embedding": emb}


def reply_assignments(arc, L: int, input_sizes: list, output_sizes: list, ops: list) -> list:
    """The two assignments of one arc [RECALL: service.py]; json.dumps turns the embedding's int keys into strings."""
    layers = organise_arc(arc, L)
    return [Assignment("architecture", json.dumps(layers).replace('"', "'")),
            Assignment("nn_config", json.dumps(nn_config(layers, L, input_sizes, output_sizes, ops)).replace('"', "'"))]


def reward_of(trials, metric_name: str):
    """Mean objective-metric value over the SUCCEEDED trials (None when there are none) [RECALL: service.py]."""
    vals = []
    for t in trials:
        if t.status.condition != api.SUCCEEDED:
            continue
        for m in t.status.observation.metrics:
            if m.name == metric_name:
                vals.append(float(m.value))
                break
    return float(np.mean(vals)) if vals else None


def _fingerprint(exp, settings: dict) -> tuple:
    return (exp.spec.nas_config.SerializeToString(deterministic=True), exp.spec.objective.objective_metric_name,
            tuple(sorted((k, repr(v)) for k, v in settings.items())))


class _EnasExperiment:
    def __init__(self, L, input_sizes, output_sizes, ops, settings):
        self.L, self.input_sizes, self.output_sizes, self.ops, self.settings = L, input_sizes, output_sizes, ops, settings
        self.seed = settings["random_state"] if "random_state" in settings else int(np.random.default_rng().integers(1 << 62))
        self.engine = None       # kubeflow_b200.enas.EnasController, created at the first call that samples
        self.calls = 0

    def close(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None


class EnasService(_Base):
    algorithm_names = (NAME,)

    def _check(self, experiment) -> tuple:
        self.check_algorithm(experiment)
        raw = parse_settings(experiment)
        settings = validate_enas_settings(raw)
        return raw, settings, parse_nas_config(experiment)

    def validate(self, experiment):
        self._check(experiment)

    def get_suggestions(self, request):
        exp = request.experiment
        raw, settings, (L, ins, outs, ops) = self._check(exp)
        settings = self.with_defaults(raw, settings)
        k = max(int(request.current_request_number), 0)
        if k > MAX_REQUEST:
            raise AlgorithmSettingsError(f"current_request_number = {k} exceeds this engine's limit of {MAX_REQUEST} arcs per call")
        if k == 0:
            return _reply_from([])
        with self._lock:
            st = self.experiment(exp.name, _fingerprint(exp, settings), lambda: _EnasExperiment(L, ins, outs, ops, settings))
            if st.engine is None:
                from ..enas import EnasController
                ctl = {k2[len("controller_"):]: settings[k2] for k2 in ("controller_temperature", "controller_tanh_const",
                                                                        "controller_entropy_weight", "controller_baseline_decay",
                                                                        "controller_learning_rate", "controller_skip_target",
                                                                        "controller_skip_weight")}
                st.engine = EnasController(L, settings["controller_hidden_size"], len(ops), settings=ctl, seed=st.seed,
                                           device=int(settings.get("device", 0)))
            R = reward_of(request.trials, exp.spec.objective.objective_metric_name)
            if st.calls > 0 and R is not None:
                stats = st.engine.train(R, settings["controller_train_steps"])
                every = settings["controller_log_every_steps"]
                for i in range(every - 1, len(stats), every):
                    logger.info("enas %s: controller step %d: loss %.6g, entropy %.6g, baseline %.6g, skip rate %.4g", exp.name,
                                i + 1, stats[i, 3], stats[i, 1], stats[i, 4], stats[i, 5])
            st.calls += 1
            arcs = st.engine.sample(k)
        return _reply_from([reply_assignments(a, L, ins, outs, ops) for a in arcs])
