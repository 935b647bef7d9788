"""``darts`` — Katib's DARTS neural-architecture search [RECALL: Katib's nas/darts/service.py].  The search itself (the
supernet, its architecture weights and their bilevel optimisation) runs inside the trial; the suggestion only hands it the
search space and the DARTS settings, as three assignments that are the same for every trial.  There is nothing for the GPU to
do here and none is used.

* ValidateAlgorithmSettings [RECALL]: ``nas_config.graph_config.num_layers`` >= 1; at least one operation; every operation other
  than ``skip_connection`` has a first parameter spec that is a non-empty CATEGORICAL list of filter sizes (further specs are
  ignored, as upstream considers only the first).  Settings are those of ``DEFAULTS``, each checked for its type and range:
  ``num_epochs``, ``init_channels``, ``print_step``, ``num_nodes`` and ``stem_multiplier`` integers >= 1, ``batch_size`` an
  integer >= 1 or ``None``, ``num_workers`` an integer >= 0, the learning rates, weight decays, ``w_momentum`` and
  ``w_grad_clip`` finite numbers >= 0.
* Reply [RECALL], ``current_request_number`` identical assignment lists:
  - ``algorithm-settings``: ``DEFAULTS`` with the Experiment's settings laid over them, each given value kept as its string;
  - ``search-space``: per operation in order, ``skip_connection`` as it is and any other ``<type>_<k>x<k>`` for each filter
    size k of its list in order;
  - ``num-layers``: the layer count in decimal.
  The first two are ``json.dumps`` text with ``"`` replaced by ``'``: trial code parses these strings, so the format is the
  contract.

Departures, all deliberate: a setting outside ``DEFAULTS`` and an operation without an ``operation_type`` are refused by name,
and no state is kept between calls (every call builds its reply from the request).
"""
from __future__ import annotations

import json
import math

from . import api_pb as api
from .internal import AlgorithmSettingsError, Assignment, parse_settings
from .service import _Base, _reply_from

NAME = "darts"
SKIP = "skip_connection"
# upstream's defaults, in upstream's order (the order of the algorithm-settings text) [RECALL]
DEFAULTS = {"num_epochs": 50, "w_lr": 0.025, "w_lr_min": 0.001, "w_momentum": 0.9, "w_weight_decay": 3e-4, "w_grad_clip": 5.0,
            "alpha_lr": 3e-4, "alpha_weight_decay": 1e-3, "batch_size": 128, "num_workers": 4, "init_channels": 16,
            "print_step": 50, "num_nodes": 4, "stem_multiplier": 3}
_INT_MIN = {"num_epochs": 1, "batch_size": 1, "num_workers": 0, "init_channels": 1, "print_step": 1, "num_nodes": 1,
            "stem_multiplier": 1}
_NONE_OK = ("batch_size",)


def validate_darts_settings(settings: dict) -> dict:
    """``DEFAULTS`` overlaid by ``settings`` (name -> value string, kept as given), or AlgorithmSettingsError naming the setting."""
    out = dict(DEFAULTS)
    for k, v in settings.items():
        if k not in DEFAULTS:
            raise AlgorithmSettingsError(f"unknown setting {k} for algorithm {NAME}")
        if not (k in _NONE_OK and v == "None"):
            try:
                x = int(v) if k in _INT_MIN else float(v)
            except ValueError:
                raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
            if k in _INT_MIN and x < _INT_MIN[k]:
                raise AlgorithmSettingsError(f"{k} should be an integer >= {_INT_MIN[k]}{' or None' if k in _NONE_OK else ''}, got {v}")
            if k not in _INT_MIN and not (math.isfinite(x) and x >= 0):
                raise AlgorithmSettingsError(f"{k} should be a number >= 0, got {v}")
        out[k] = v
    return out


def search_space(operations) -> list:
    """The operation names of the search space, or AlgorithmSettingsError naming the operation [RECALL: get_search_space]."""
    out = []
    for op in operations:
        if not op.operation_type:
            raise AlgorithmSettingsError("nas_config: every operation needs an operation_type")
        if op.operation_type == SKIP:
            out.append(SKIP)
            continue
        specs = list(op.parameter_specs.parameters)
        if not specs or specs[0].parameter_type != api.CATEGORICAL or not len(specs[0].feasible_space.list):
            raise AlgorithmSettingsError(f"nas_config: operation {op.operation_type!r} needs a first parameter spec that is a "
                                         f"non-empty CATEGORICAL list of filter sizes")
        out.extend(f"{op.operation_type}_{k}x{k}" for k in specs[0].feasible_space.list)
    if not out:
        raise AlgorithmSettingsError("nas_config needs at least one operation")
    return out


def reply_assignments(experiment) -> list:
    """The three assignments every trial of ``experiment`` gets, or AlgorithmSettingsError."""
    nc = experiment.spec.nas_config
    L = int(nc.graph_config.num_layers)
    if L < 1:
        raise AlgorithmSettingsError(f"nas_config: graph_config.num_layers must be >= 1, got {L}")
    ops = search_space(nc.operations.operation)
    settings = validate_darts_settings(parse_settings(experiment))
    return [Assignment("algorithm-settings", json.dumps(settings).replace('"', "'")),
            Assignment("search-space", json.dumps(ops).replace('"', "'")),
            Assignment("num-layers", str(L))]


class DartsService(_Base):
    algorithm_names = (NAME,)

    def validate(self, experiment):
        self.check_algorithm(experiment)
        reply_assignments(experiment)

    def get_suggestions(self, request):
        self.check_algorithm(request.experiment)
        assignments = reply_assignments(request.experiment)
        return _reply_from([assignments] * max(int(request.current_request_number), 0))
