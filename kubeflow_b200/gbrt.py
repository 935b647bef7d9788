"""GBRT on the GPU (libkbo ``kbo_gbrt_*``) — skopt's ``GradientBoostingQuantileRegressor`` surrogate, the estimator skopt's
``cook_estimator("GBRT")`` builds: three ``GradientBoostingRegressor(loss="quantile", n_estimators=30)`` chains at α = 0.16, 0.5
and 0.84, fitted together on the device; ``predict(return_std=True)`` gives the middle chain as the mean and half the spread of the
outer two as the standard deviation, negative where the quantiles cross (FP64 restatement: oracle/gbrt_oracle.py).

Like the forests, the trees are built on the transformed [0, 1] coordinates the rest of the engine uses, where skopt builds on the
raw parameter values: the map is affine per column, so the trees have the same structure up to sklearn's 1e-7 feature threshold.
Exact ties between splits go to the lowest feature (sklearn visits features in a random order), and a node whose rows all lie on
one side of the current prediction is a leaf (sklearn may split it on rounding noise in its impurity).

Pass an instance to ``Optimizer(base_estimator=GbrtEngine(...))``, the way skopt's ``gbrt_minimize`` passes a
``GradientBoostingQuantileRegressor``: the string ``"GBRT"`` is not accepted there.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .tree import TreeEngine

SKOPT_QUANTILES = (0.16, 0.5, 0.84)


class GbrtEngine(TreeEngine):
    _SWEEP_TAIL = (None,)          # quantiles_out

    def __init__(self, device: int = 0, *, quantiles=SKOPT_QUANTILES, n_estimators: int = 30, acq: str = "ei", xi: float = 0.01,
                 kappa: float = 1.96):
        q = tuple(float(v) for v in quantiles)
        if len(q) != 3:
            raise ValueError(f"quantiles must hold three values (lower, middle, upper), got {quantiles!r}")
        self.quantiles, self.n_estimators = q, int(n_estimators)
        super().__init__(device, "gbrt", ((C.c_double * 3)(*q), self.n_estimators), acq, xi, kappa)

    def _fit(self, Xd, yd, N, D, counts):
        return self.lib.kbo_gbrt_fit(self._h, self._o, Xd.data_ptr(), yd.data_ptr(), N, D, self._stream())

    def predict(self, X, return_std: bool = False, return_quantiles: bool = False):
        """skopt's predict: the mean (float64 NumPy) at the rows of X; with ``return_std`` also the standard deviation; with
        ``return_quantiles`` the 3 × n chain predictions (lower, middle, upper) instead."""
        Xh = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float32)))
        self._check(Xh.shape[1])
        n = len(Xh)
        mu, sd, q = np.empty(n), np.empty(n), np.empty((3, n))
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_gbrt_predict(self._h, self._o, Xh.ctypes.data, n, 1, mu.ctypes.data, sd.ctypes.data, q.ctypes.data,
                                                 self._stream()))
        if return_quantiles:
            return q
        return (mu, sd) if return_std else mu

    def predict_mean(self, X) -> np.ndarray:
        return self.predict(X)

    def export(self, chain: int, stage: int) -> dict:
        """The tree of stage ``stage`` of chain ``chain`` (0: lower, 1: middle, 2: upper quantile) in sklearn's ``tree_`` layout
        (depth-first preorder), with ``n_pos`` (rows with y >= raw at that stage) and the chain's ``init``."""
        n, init = C.c_int32(), C.c_double()
        self.check(self.lib.kbo_gbrt_export(self._h, self._o, int(chain), int(stage), *([None] * 7), 0, C.byref(n), C.byref(init),
                                            self._stream()))
        k = n.value
        out = dict(feature=np.empty(k, np.int32), threshold=np.empty(k), left=np.empty(k, np.int32), right=np.empty(k, np.int32),
                   value=np.empty(k), n_node_samples=np.empty(k, np.int32), n_pos=np.empty(k, np.int32))
        self.check(self.lib.kbo_gbrt_export(
            self._h, self._o, int(chain), int(stage),
            *[out[a].ctypes.data for a in ("feature", "threshold", "left", "right", "value", "n_node_samples", "n_pos")], k, None, None,
            self._stream()))
        out["init"] = init.value
        return out
