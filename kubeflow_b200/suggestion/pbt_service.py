"""``pbt`` — Population Based Training (Jaderberg et al., "Population Based Training of Neural Networks", 2017), served under
Katib's algorithm name.  Katib's own PBT service is not available here; its rules are restated from memory and marked [RECALL],
and where memory and the paper disagree the paper's defaults are followed.  The contract is ``oracle/pbt_oracle.py``, an
independent plain-Python restatement of one call that the service must match decision for decision on the same draws.

This is host-side bookkeeping by nature (a sort of at most a few hundred objective values and a handful of draws per call); there
is nothing for the GPU to do here and none is used.

* Settings [RECALL]: ``suggestion_trial_dir`` (required, an absolute path: the root of the per-trial checkpoint directories on the
  volume the suggestion pod shares with the trials), ``n_population`` (int >= 5, default 40), ``truncation_threshold`` (float in
  (0, 1), default 0.2), ``resample_probability`` (float in [0, 1]; unset: always perturb, never resample), ``random_state``.
  Parameters may be DOUBLE, INT, DISCRETE or CATEGORICAL.
* Population.  Each trial takes over one of ``n_population`` slots from its *predecessor* (the slot's previous trial).  A slot's
  member is its latest completed trial (SUCCEEDED or EARLYSTOPPED, with the objective metric): the current trial if it has
  completed, else, while the current trial runs, its predecessor, unless the running trial is a fresh start.  A slot whose current
  trial ended otherwise (FAILED, KILLED, METRICSUNAVAILABLE, or no usable metric) has no member: its lineage has ended.
* Generation 0: ``n_population`` prior draws, one slot each; they come first, so a population larger than the Experiment's
  parallelism fills before any lineage advances.  Prior draws are uniform like ``random``'s (one uniform per parameter value).
* Exploit (truncation selection [RECALL], the paper's defaults): members rank by objective, best first (MINIMIZE ascending,
  MAXIMIZE descending; ties: lower generation first, then trial name).  With n members, n_cut = ⌊threshold·n⌋ (plus 1e-9 against
  rounding).  A completed member whose rank is among the last n_cut hands its slot to a child of a member drawn uniformly from
  the first n_cut (the *parent*: the child copies its hyperparameters and checkpoint); any other completed member continues its
  own lineage with the same hyperparameters (it is its own parent).  Above a threshold of 0.5 the two ends overlap and a member
  may draw itself.  A slot whose lineage ended gets a fresh prior draw (no parent), so the population stays at ``n_population``.
* Explore, on exploited children only (the paper): per parameter in spec order, with probability ``resample_probability`` a prior
  redraw; otherwise DOUBLE and INT values are multiplied by 0.8 or 1.2 (even odds); INT values are then rounded half up, and
  if that leaves the value unchanged it steps by 1 in the direction the factor moved it (up for 1.2 and down for 0.8 at 0); the
  result is clipped to [min, max].  DISCRETE and CATEGORICAL values move to the previous or next list entry (even odds), clamped at
  the ends.  The list-neighbour rule and the INT step are this engine's choices.
* Which slots are served: a call returns up to ``current_request_number`` trials, fewer when fewer slots are free [RECALL]:
  missing generation-0 slots first, then slots whose current trial has finished, lowest generation first, then by name (so no
  lineage waits behind the others when the Experiment's parallelism is below ``n_population``).
* Reply: each trial is named by the service [RECALL]: the experiment name (lower-cased, characters outside [a-z0-9-] replaced by
  ``-``, at most 54 characters, no leading or trailing ``-``), ``-`` and 8 lowercase alphanumerics, a DNS-1123 label of at most
  63 characters.  Labels: ``pbt.suggestion.katib.kubeflow.org/generation`` (the parent's generation + 1; 0 without a parent) and
  ``.../parent`` (omitted for prior draws) [RECALL], and ``.../predecessor``, the trial whose slot it takes (omitted for
  generation 0).  The predecessor label is this engine's addition: an exploited child's parent is the top member it copies, so
  the two recalled labels cannot tell which member it replaced, and the population could not be rebuilt from the trials.
* Checkpoint hand-off [RECALL]: before the reply, ``suggestion_trial_dir/<child>`` is made a copy of ``suggestion_trial_dir/<parent>``
  (an existing ``<child>`` entry is replaced, so a re-issued name gets the same copy).  A parent without a directory, and a prior
  draw, get an empty directory (the former is logged).  Trial names must be DNS-1123 subdomains, so no name resolves outside
  ``suggestion_trial_dir``; a request with any other name is refused.
* State: every call rebuilds the population from ``request.trials`` (Katib sends every trial of the Experiment, running ones
  included, with the labels above), so a restarted service continues the same Experiment.  Draws come from a Generator seeded by
  (random_state, experiment name, the sorted names of every known trial), never from a running generator.  The one in-process
  state is the record of names issued and not yet seen in ``request.trials``, per experiment under a lock, so that a repeated
  call does not serve those slots twice; a name leaves the record when its trial arrives.
* Every draw is one ``rng.random()`` uniform, taken in this order per issued trial: the parent pick (exploit), per parameter the
  resample test (when ``resample_probability`` is set) and the redraw or perturbation (exploit) or the prior draw (fresh), then
  8 for the name (again 8 on the rare collision with a known name).
"""
from __future__ import annotations

import hashlib
import logging
import math
import os
import re
import shutil
import threading
from dataclasses import dataclass, field

import numpy as np

from . import api_pb as api
from .internal import (DOUBLE, INTEGER, MAX_GOAL, AlgorithmSettingsError, Assignment, HyperParameterSearchSpace, Trial,
                       parse_settings)
from .service import _Base, _reply_from, experiment_fingerprint

logger = logging.getLogger(__name__)

NAME = "pbt"
LABEL_PREFIX = "pbt.suggestion.katib.kubeflow.org/"
GENERATION, PARENT, PREDECESSOR = LABEL_PREFIX + "generation", LABEL_PREFIX + "parent", LABEL_PREFIX + "predecessor"
DEFAULTS = dict(n_population=40, truncation_threshold=0.2, resample_probability=None)
NAME_ALPHABET = "abcdefghijklmnopqrstuvwxyz0123456789"
_SUBDOMAIN = re.compile(r"[a-z0-9]([-a-z0-9]*[a-z0-9])?(\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*")

IN_FLIGHT, COMPLETED, ENDED = "in flight", "completed", "ended"
_FINISHED = (api.SUCCEEDED, api.EARLYSTOPPED, api.FAILED, api.KILLED, api.METRICSUNAVAILABLE)


def validate_pbt_settings(settings: dict) -> dict:
    """Parsed settings with defaults, or AlgorithmSettingsError naming the setting."""
    out = dict(DEFAULTS)
    for k, v in settings.items():
        try:
            if k == "suggestion_trial_dir":
                x = str(v)
                if not os.path.isabs(x):
                    raise AlgorithmSettingsError(f"suggestion_trial_dir should be an absolute path, got {v!r}")
            elif k == "n_population":
                x = int(v)
                if x < 5:
                    raise AlgorithmSettingsError(f"n_population should be an integer >= 5, got {v}")
            elif k == "truncation_threshold":
                x = float(v)
                if not 0.0 < x < 1.0:
                    raise AlgorithmSettingsError(f"truncation_threshold should be in (0, 1), got {v}")
            elif k == "resample_probability":
                x = float(v)
                if not 0.0 <= x <= 1.0:
                    raise AlgorithmSettingsError(f"resample_probability should be in [0, 1], got {v}")
            elif k == "random_state":
                x = int(v)
                if x < 0:
                    raise AlgorithmSettingsError(f"random_state should be great or equal than zero, got {v}")
            else:
                raise AlgorithmSettingsError(f"unknown setting {k} for algorithm {NAME}")
            out[k] = x
        except AlgorithmSettingsError:
            raise
        except (TypeError, ValueError):
            raise AlgorithmSettingsError(f"failed to convert {v!r} for setting {k}")
    if "suggestion_trial_dir" not in out:
        raise AlgorithmSettingsError(f"suggestion_trial_dir must be set for {NAME}")
    return out


@dataclass
class PbtTrial:
    name: str
    generation: int
    parent: str | None
    predecessor: str | None
    values: dict                      # parameter name -> value string
    objective: float | None = None
    state: str = IN_FLIGHT

    def labels(self) -> dict:
        out = {GENERATION: str(self.generation)}
        if self.parent:
            out[PARENT] = self.parent
        if self.predecessor:
            out[PREDECESSOR] = self.predecessor
        return out


def parse_trials(trials) -> list:
    """The request's trials as PbtTrial, refusing names that are not DNS-1123 subdomains (they name directories)."""
    objectives = {}
    for t in Trial.convert(trials):
        try:
            y = float(t.target_metric.value)
        except ValueError:
            continue
        if not math.isnan(y):
            objectives[t.name] = y
    out = []
    for t in trials:
        if len(t.name) > 253 or not _SUBDOMAIN.fullmatch(t.name):
            raise AlgorithmSettingsError(f"trial name {t.name!r} is not a DNS-1123 subdomain, so it cannot name a directory "
                                         f"under suggestion_trial_dir")
        labels = t.spec.labels
        try:
            gen = int(labels.get(GENERATION, "0"))
        except ValueError:
            raise AlgorithmSettingsError(f"trial {t.name}: label {GENERATION} = {labels.get(GENERATION)!r} is not an integer")
        if t.status.condition in (api.SUCCEEDED, api.EARLYSTOPPED) and t.name in objectives:
            state = COMPLETED
        else:
            state = ENDED if t.status.condition in _FINISHED else IN_FLIGHT
        out.append(PbtTrial(t.name, gen, labels.get(PARENT) or None, labels.get(PREDECESSOR) or None,
                            {a.name: a.value for a in t.spec.parameter_assignments.assignments}, objectives.get(t.name), state))
    return out


def call_rng(random_state, experiment: str, names):
    """The Generator of one call: seeded by (random_state, experiment name, sorted trial names); fresh entropy without a
    random_state."""
    if random_state is None:
        return np.random.default_rng()
    h = hashlib.sha256("\n".join([experiment, *sorted(names)]).encode()).digest()
    return np.random.default_rng([int(random_state), *np.frombuffer(h, dtype="<u4").tolist()])


def _prior_value(p, u: float) -> str:
    if p.type == DOUBLE:
        lo, hi = float(p.min), float(p.max)
        return repr(lo + u * (hi - lo))
    if p.type == INTEGER:
        lo, hi = int(p.min), int(p.max)
        return str(min(lo + int(u * (hi - lo + 1)), hi))
    return p.list[min(int(u * len(p.list)), len(p.list) - 1)]


def _perturb(p, value: str, u: float) -> str:
    if p.type in (DOUBLE, INTEGER):
        f = 0.8 if u < 0.5 else 1.2
        if p.type == DOUBLE:
            return repr(min(max(float(value) * f, float(p.min)), float(p.max)))
        v = int(value)
        x = math.floor(v * f + 0.5)
        if x == v:
            x = v + (1 if (f > 1.0) == (v >= 0) else -1)
        return str(min(max(x, int(p.min)), int(p.max)))
    if value not in p.list:
        raise ValueError(f"parameter {p.name!r}: value {value!r} is not in its feasible list")
    i = p.list.index(value) + (-1 if u < 0.5 else 1)
    return p.list[min(max(i, 0), len(p.list) - 1)]


def _trial_name(experiment: str, rng, taken) -> str:
    prefix = re.sub(r"[^a-z0-9-]", "-", experiment.lower())[:54].strip("-")
    while True:
        tail = "".join(NAME_ALPHABET[min(int(rng.random() * 36), 35)] for _ in range(8))
        name = f"{prefix}-{tail}" if prefix else tail
        if name not in taken:
            return name


def plan(trials: list, ss, settings: dict, rng, k: int, experiment: str) -> list:
    """The next (up to k) trials, as in-flight PbtTrials, for the known trials (the request's plus those issued and not yet
    seen); draws from ``rng.random()`` only."""
    by_name = {t.name: t for t in trials}
    superseded = {t.predecessor for t in trials if t.predecessor}
    current = [t for t in trials if t.name not in superseded]
    members = []
    for t in current:
        if t.state == COMPLETED:
            members.append(t)
        elif t.state == IN_FLIGHT and t.parent and t.predecessor in by_name and by_name[t.predecessor].state == COMPLETED:
            members.append(by_name[t.predecessor])
    sign = -1.0 if ss.goal == MAX_GOAL else 1.0
    ranked = sorted(members, key=lambda t: (sign * t.objective, t.generation, t.name))
    rank = {t.name: i for i, t in enumerate(ranked)}
    n_cut = int(math.floor(settings["truncation_threshold"] * len(ranked) + 1e-9))
    n_roots = sum(1 for t in trials if not t.predecessor)
    free = [None] * max(settings["n_population"] - n_roots, 0)
    free += sorted((t for t in current if t.state != IN_FLIGHT), key=lambda t: (t.generation, t.name))
    taken, out = set(by_name), []
    for slot in free[:max(k, 0)]:
        if slot is None or slot.state == ENDED:
            parent, values = None, {p.name: _prior_value(p, rng.random()) for p in ss.params}
        elif rank[slot.name] < len(ranked) - n_cut:
            parent, values = slot, {p.name: _value_of(slot, p) for p in ss.params}
        else:
            parent = ranked[min(int(rng.random() * n_cut), n_cut - 1)]
            values, p_re = {}, settings["resample_probability"]
            for p in ss.params:
                if p_re is not None and rng.random() < p_re:
                    values[p.name] = _prior_value(p, rng.random())
                else:
                    values[p.name] = _perturb(p, _value_of(parent, p), rng.random())
        name = _trial_name(experiment, rng, taken)
        taken.add(name)
        out.append(PbtTrial(name, parent.generation + 1 if parent else 0, parent.name if parent else None,
                            slot.name if slot else None, values))
    return out


def _value_of(t: PbtTrial, p) -> str:
    if p.name not in t.values:
        raise ValueError(f"trial {t.name} has no assignment for parameter {p.name!r}")
    return t.values[p.name]


def hand_off(root: str, parent: str | None, child: str):
    """Makes ``root/child`` a copy of ``root/parent`` (an empty directory without one); both are single path components."""
    dst = os.path.join(root, child)
    if os.path.islink(dst) or os.path.isfile(dst):
        os.unlink(dst)
    elif os.path.isdir(dst):
        shutil.rmtree(dst)
    src = os.path.join(root, parent) if parent else None
    if src is not None and os.path.isdir(src):
        shutil.copytree(src, dst, symlinks=True)
        return
    if src is not None:
        logger.info("pbt: parent %s has no directory under %s; %s starts from an empty one", parent, root, child)
    os.mkdir(dst)


@dataclass
class _PbtExperiment:
    lock: threading.Lock = field(default_factory=threading.Lock)
    issued: dict = field(default_factory=dict)    # name -> PbtTrial handed out and not yet seen in request.trials

    def close(self):
        pass


class PbtService(_Base):
    algorithm_names = (NAME,)
    MAX_EXPERIMENTS = 64          # an entry is a few issued names, no device memory

    def _check(self, experiment) -> tuple:
        self.check_algorithm(experiment)
        return HyperParameterSearchSpace.convert(experiment), validate_pbt_settings(parse_settings(experiment))

    def validate(self, experiment):
        self._check(experiment)

    def get_suggestions(self, request):
        exp = request.experiment
        ss, st = self._check(exp)
        k = max(int(request.current_request_number), 0)
        trials = parse_trials(request.trials)
        if k == 0:
            return _reply_from([])
        root = st["suggestion_trial_dir"]
        if not os.path.isdir(root):
            raise AlgorithmSettingsError(f"suggestion_trial_dir {root} is not a directory")
        with self._lock:
            entry = self.experiment(exp.name, experiment_fingerprint(exp, ss, st), _PbtExperiment)
        with entry.lock:
            for t in trials:
                entry.issued.pop(t.name, None)
            known = trials + list(entry.issued.values())
            picks = plan(known, ss, st, call_rng(st.get("random_state"), exp.name, [t.name for t in known]), k, exp.name)
            for t in picks:
                hand_off(root, t.parent, t.name)
            entry.issued.update((t.name, t) for t in picks)
        logger.info("pbt %s: %d known trials, %d requested, %d issued", exp.name, len(known), k, len(picks))
        reply = _reply_from([[Assignment(p.name, t.values[p.name]) for p in ss.params] for t in picks])
        for pa, t in zip(reply.parameter_assignments, picks):
            pa.trial_name = t.name
            pa.labels.update(t.labels())
        return reply
