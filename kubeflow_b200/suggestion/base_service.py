"""``BaseSkoptService`` — mirror of kubeflow/katib pkg/suggestion/v1beta1/skopt/base_service.py: holds the
optimizer for one experiment, tells it the trials it has not seen yet and asks for ``current_request_number``
new assignments (SURVEY.md §3.1)."""
from __future__ import annotations

import logging

from ..optimizer import Optimizer
from ..space import Categorical, Integer, Real
from .internal import DOUBLE, INTEGER, MAX_GOAL, Assignment

logger = logging.getLogger(__name__)


def dimensions(search_space) -> list:
    """The ``Space`` dimensions of a Katib search space: INT → Integer, DOUBLE → Real, CATEGORICAL / DISCRETE → Categorical."""
    return [Integer(int(p.min), int(p.max), name=p.name) if p.type == INTEGER else
            Real(float(p.min), float(p.max), name=p.name) if p.type == DOUBLE else Categorical(list(p.list), name=p.name)
            for p in search_space.params]


class BaseSkoptService:
    def __init__(self, base_estimator="GP", n_initial_points=10, acq_func="gp_hedge", acq_optimizer="auto", random_state=None,
                 search_space=None, **engine_settings):
        self.base_estimator, self.n_initial_points = base_estimator, n_initial_points
        self.acq_func, self.acq_optimizer, self.random_state = acq_func, acq_optimizer, random_state
        self.search_space = search_space
        self.engine_settings = engine_settings
        self.skopt_optimizer = None
        self.told_trials = set()
        self._told_hashes = set()     # kbo_hash64 of the told names: the request scan compares hashes, not strings
        self.create_optimizer()

    def create_optimizer(self):
        self.skopt_optimizer = Optimizer(dimensions(self.search_space), base_estimator=self.base_estimator, n_initial_points=self.n_initial_points,
                                         acq_func=self.acq_func, acq_optimizer=self.acq_optimizer, random_state=self.random_state,
                                         **self.engine_settings)

    def close(self):
        self.skopt_optimizer.close()

    def getSuggestions(self, trials, current_request_number):
        """trials: internal.Trial list (all completed trials, resent every call); returns a list of Assignment lists."""
        skopt_suggested, loss_for_skopt, new_names = [], [], []
        for trial in trials:
            if trial.name in self.told_trials or trial.name in new_names:
                continue
            row = []
            by_name = {a.name: a.value for a in trial.assignments}
            for param in self.search_space.params:
                value = by_name.get(param.name)
                if value is None:
                    raise ValueError(f"trial {trial.name!r} has no assignment for parameter {param.name!r}")
                row.append(int(value) if param.type == INTEGER else float(value) if param.type == DOUBLE else value)
            loss = float(trial.target_metric.value)
            if self.search_space.goal == MAX_GOAL:
                loss = -1.0 * loss
            skopt_suggested.append(row)
            loss_for_skopt.append(loss)
            new_names.append(trial.name)
        if skopt_suggested:
            self.skopt_optimizer.tell(skopt_suggested, loss_for_skopt)
            self.told_trials.update(new_names)   # only once tell() succeeded: a bad later trial must not mark earlier ones as told
        points = self.skopt_optimizer.ask(n_points=current_request_number)
        return [self.convert(self.search_space, p) for p in points]

    def ingest(self, request) -> bool:
        """Fast equivalent of the loop above for a ``LazyRequest``: tells the optimizer every usable trial it has not seen,
        straight from the request scan's arrays.  Returns False — having told nothing — whenever a new trial needs the
        reference's own conversion or error path (a value that is not a plain decimal literal, a missing assignment, an
        objective that is not a number): the caller then walks the parsed messages as before."""
        import numpy as np
        from .ingest import MISSING, hash64
        params = self.search_space.params
        if len(self._told_hashes) != len(self.told_trials):       # names told through the message path: hash them once
            self._told_hashes = {hash64(n) for n in self.told_trials}
        head = request.trial_table([])                            # names, conditions, objective: no numbers parsed yet
        told = np.fromiter(self._told_hashes, dtype=np.uint64, count=len(self._told_hashes))
        idx = np.flatnonzero(head.usable & ~np.isin(head.name_hash, told))
        if idx.size:
            _, first = np.unique(head.name_hash[idx], return_index=True)  # a name sent twice in one request is told once
            idx = idx[np.sort(first)]
        if idx.size == 0:
            return True
        mask = np.zeros(head.n, dtype=bool)
        mask[idx] = True
        tab = request.trial_table([p.name for p in params], select=mask)   # assignments of the new trials only
        flags, lens = tab.value_flags[idx], tab.value_len[idx]
        if not (tab.objective_flags[idx] & 1).all() or (lens == MISSING).any():
            return False
        num_cols = [j for j, p in enumerate(params) if p.type in (INTEGER, DOUBLE)]
        for j in num_cols:
            if not (flags[:, j] & (2 if params[j].type == INTEGER else 1)).all():
                return False
        names = [request.text(tab.name_off[i], tab.name_len[i]) for i in idx]
        vals = tab.values[idx]
        cols, xt_cols = [], []
        for j, (p, dim) in enumerate(zip(params, self.skopt_optimizer.space.dimensions)):
            if p.type == INTEGER:
                iv = vals[:, j].astype(np.int64)
                cols.append(iv.tolist())
                xt_cols.append(((iv - int(dim.low)).astype(np.float64) / float(dim.high - dim.low))[:, None])
            elif p.type == DOUBLE:
                cols.append(vals[:, j].tolist())
                xt_cols.append(((vals[:, j] - dim.low) / (dim.high - dim.low))[:, None])
            else:
                sv = [request.text(tab.value_off[i, j], tab.value_len[i, j]) for i in idx]
                cols.append(sv)
                xt_cols.append(np.asarray([dim.to_unit(v) for v in sv], dtype=np.float64).reshape(len(sv), dim.width))
        rows = [list(r) for r in zip(*cols)]
        loss = tab.objective[idx]
        if self.search_space.goal == MAX_GOAL:
            loss = -1.0 * loss
        self.skopt_optimizer.tell(rows, loss.tolist(), xt=np.concatenate(xt_cols, axis=1))
        self.told_trials.update(names)
        self._told_hashes.update(int(h) for h in tab.name_hash[idx])
        return True

    @staticmethod
    def convert(search_space, skopt_suggested):
        out = []
        for param, v in zip(search_space.params, skopt_suggested):
            if param.type == INTEGER:
                out.append(Assignment(param.name, str(int(v))))
            elif param.type == DOUBLE:
                out.append(Assignment(param.name, repr(float(v))))
            else:
                out.append(Assignment(param.name, str(v)))
        return out
