"""``multivariate-tpe`` — Katib's Optuna-backed multivariate Tree-structured Parzen Estimator on the GPU engine
``kubeflow_b200.mvtpe`` (contract: oracle/mvtpe_oracle.py, whose docstring lists every recalled detail; parity with Optuna and
Katib's Optuna service is unpinned).

* Space: DOUBLE → float on [min, max]; INT → integers min, min + q, ... <= max, q = ``step`` or 1, reported as integers;
  CATEGORICAL / DISCRETE → categorical over the list, observed as the category index.
* History: the usable trials (``Trial.convert``), each told once by name, kept in the order first told; loss = objective value,
  negated for MAXIMIZE.  A trial whose objective is NaN is never told (Optuna fails such trials); ±inf are ranked.
* While fewer than ``n_startup_trials`` trials are told, points come from independent uniform sampling — the sampling
  ``random`` uses — and no GPU handle exists.  Then every point is the best of ``n_ei_candidates`` candidate vectors drawn
  from the joint below model and scored on the device.
* Batches (``current_request_number`` = k > 1): k independent draws against the same model, with no lies in between, as k
  calls of Optuna's ``study.ask`` with the pending trials ignored.
* Draws are keyed by (random_state, ask counter, point, candidate, slot): the same request sequence gives the same replies.
* Under the SPMD server every rank scores its block of each request's candidates, as for ``tpe`` (tpe_service.py).
"""
from __future__ import annotations

import numpy as np

from .internal import DOUBLE, INTEGER, AlgorithmSettingsError, HyperParameterSearchSpace, parse_settings
from .service import _Base, _reply_from, experiment_fingerprint
from .tpe_service import _Experiment, sharded_points

NAME = "multivariate-tpe"
MAX_EI_CANDIDATES = 1 << 24
MAX_PARAMETERS = 65535            # kbo_mvtpe_create's limit on D


def validate_mvtpe_settings(settings: dict) -> dict:
    """Parsed settings with defaults, or AlgorithmSettingsError naming the setting [RECALL: Katib's Optuna validation]."""
    out = dict(n_startup_trials=10, n_ei_candidates=24)
    for k, v in settings.items():
        try:
            if k == "n_startup_trials":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"n_startup_trials should be greater or equal than zero, got {v}")
            elif k == "n_ei_candidates":
                out[k] = int(v)
                if not 1 <= out[k] <= MAX_EI_CANDIDATES:
                    raise AlgorithmSettingsError(f"n_ei_candidates should be in [1, 2^24], got {v}")
            elif k == "random_state":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"random_state should be greater or equal than zero, got {v}")
            elif k == "device":
                out[k] = int(v)
                if out[k] < 0:
                    raise AlgorithmSettingsError(f"device should be greater or equal than zero, got {v}")
            else:
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm {NAME}")
        except AlgorithmSettingsError:
            raise
        except (TypeError, ValueError):
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
    return out


def mvtpe_space(ss) -> list:
    """The engine's parameter list for a Katib search space."""
    if len(ss.params) > MAX_PARAMETERS:
        raise AlgorithmSettingsError(f"{NAME} supports at most {MAX_PARAMETERS} parameters, got {len(ss.params)}")
    out = []
    for p in ss.params:
        if p.type == DOUBLE:
            lo, hi = float(p.min), float(p.max)
            if not (np.isfinite(lo) and np.isfinite(hi) and lo < hi):
                raise AlgorithmSettingsError(f"parameter {p.name!r}: {NAME} needs finite min < max, got [{p.min}, {p.max}]")
            out.append(("float", lo, hi))
        elif p.type == INTEGER:
            q = float(p.step) if p.step else 1.0
            if not q > 0:
                raise AlgorithmSettingsError(f"parameter {p.name!r}: step must be > 0, got {p.step}")
            lo, hi = float(p.min), float(p.max)
            if not lo <= hi or (hi - lo) / q >= 2 ** 31 - 2:
                raise AlgorithmSettingsError(f"parameter {p.name!r}: need min <= max and fewer than 2^31 - 1 levels")
            out.append(("int", lo, hi, q))
        else:
            out.append(("cat", len(p.list)))
    return out


class _MvExperiment(_Experiment):
    def __init__(self, ss, settings):
        super().__init__(ss, settings)
        self.space = mvtpe_space(ss)

    def row(self, trial) -> list:
        """As ``tpe``'s, with integers taken to their nearest grid point (the start-up sampler draws every integer in
        [min, max]) and floats required to lie in [min, max]."""
        row = super().row(trial)
        for d, (p, s) in enumerate(zip(self.ss.params, self.space)):
            if s[0] == "int":
                last = int(np.floor((s[2] - s[1]) / s[3]))
                row[d] = s[1] + min(max(int(np.round((row[d] - s[1]) / s[3])), 0), last) * s[3]
            elif s[0] == "float" and not s[1] <= row[d] <= s[2]:
                raise ValueError(f"trial {trial.name!r}: {row[d]!r} is outside the range of {p.name!r}")
        return row


class MultivariateTpeService(_Base):
    algorithm_names = (NAME,)

    def validate(self, experiment):
        self.check_algorithm(experiment)
        mvtpe_space(HyperParameterSearchSpace.convert(experiment))
        validate_mvtpe_settings(parse_settings(experiment))

    def get_suggestions(self, request):
        exp = request.experiment
        self.check_algorithm(exp)
        ss = HyperParameterSearchSpace.convert(exp)
        mvtpe_space(ss)
        raw = parse_settings(exp)
        settings = self.with_defaults(raw, validate_mvtpe_settings(raw))
        k = max(int(request.current_request_number), 0)
        with self._lock:
            st = self.experiment(exp.name, experiment_fingerprint(exp, ss, settings), lambda: _MvExperiment(ss, settings))
            st.ingest(request.trials, ss.goal, skip_nan=True)      # a NaN objective is a failed trial in Optuna: never told

            def make_engine():
                from ..mvtpe import MvTpe
                return MvTpe(st.space, seed=st.seed, device=int(settings.get("device", 0)))
            return _reply_from(sharded_points(self, exp.name, st, k, settings["n_startup_trials"], settings["n_ei_candidates"], make_engine))
