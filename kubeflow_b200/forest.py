"""Tree forests on the GPU (libkbo ``kbo_forest_*``) — the surrogates behind ``bayesianoptimization`` with ``base_estimator``
RF or ET: skopt's ``cook_estimator`` forests, ``RandomForestRegressor(n_estimators=100, min_samples_leaf=3)`` and
``ExtraTreesRegressor(n_estimators=100, min_samples_leaf=3)``, with skopt's ``_return_std`` and EI / LCB / PI on the raw mean
and standard deviation (FP64 restatement: oracle/forest_oracle.py).

Two deliberate differences from skopt:

* the trees are built on the transformed [0, 1] coordinates the rest of the engine uses, where skopt builds on the raw
  parameter values.  The map is affine per column, so the trees have the same structure — except that sklearn never splits a
  feature whose values lie within 1e-7 of each other (FEATURE_THRESHOLD), which a raw range narrower than 1e-7 always does and a
  transformed one does not;
* bootstrap samples and ET thresholds come from the built-in Philox stream (``kbo.h``), not NumPy's RandomState: the forests
  match sklearn's in distribution, and bit for bit once the draws are fixed (``fit(counts=...)``).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .tree import TreeEngine

KINDS = {"RF": 0, "ET": 1}


class ForestEngine(TreeEngine):
    def __init__(self, device: int = 0, *, kind: str = "RF", n_trees: int = 100, min_samples_leaf: int = 3, seed: int = 0,
                 acq: str = "ei", xi: float = 0.01, kappa: float = 1.96):
        if kind not in KINDS:
            raise ValueError(f"kind must be RF or ET, got {kind!r}")
        self.kind, self.n_trees = kind, int(n_trees)
        super().__init__(device, "forest", (KINDS[kind], self.n_trees, int(min_samples_leaf), int(seed) & (2 ** 64 - 1)), acq, xi, kappa)

    def tell(self, X, y, counts=None):
        """Fit the forest to (X, y): X in the transformed space (cast to float32, as sklearn does), y minimised.  The forest is
        kept when X and y equal the last fit's.  ``counts``: optional T × N bootstrap counts (RF) replacing the drawn ones."""
        self._tell(X, y, counts)

    def _fit(self, Xd, yd, N, D, counts):
        cd = None
        if counts is not None:
            cd = torch.from_numpy(np.ascontiguousarray(counts, dtype=np.int32).reshape(self.n_trees, N)).to(f"cuda:{self.device}")
        return self.lib.kbo_forest_fit(self._h, self._o, Xd.data_ptr(), yd.data_ptr(), N, D, cd.data_ptr() if cd is not None else None,
                                       self._stream())

    def predict(self, X):
        """(mu, sigma) float64 NumPy arrays at the rows of X: skopt's forest predict(return_std=True)."""
        Xh = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float32)))
        self._check(Xh.shape[1])
        mu, sd = np.empty(len(Xh)), np.empty(len(Xh))
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_forest_predict(self._h, self._o, Xh.ctypes.data, len(Xh), 1, mu.ctypes.data, sd.ctypes.data,
                                                   self._stream()))
        return mu, sd

    def predict_mean(self, X) -> np.ndarray:
        return self.predict(X)[0]

    def export(self, tree: int, with_draws: bool = False) -> dict:
        """Tree ``tree`` in sklearn's ``tree_`` layout (breadth-first node ids), with its bootstrap counts; ``with_draws`` (ET): the
        n_nodes × D thresholds drawn at each internal node (NaN where the feature is constant there)."""
        n = C.c_int32()
        counts = np.zeros(self.N, np.int32)
        self.check(self.lib.kbo_forest_export(self._h, self._o, int(tree), *([None] * 9), 0, C.byref(n), counts.ctypes.data,
                                              self._stream()))
        k = n.value
        out = dict(feature=np.empty(k, np.int32), threshold=np.empty(k), left=np.empty(k, np.int32), right=np.empty(k, np.int32),
                   value=np.empty(k), impurity=np.empty(k), n_node_samples=np.empty(k, np.int32), weighted_n_node_samples=np.empty(k))
        draws = np.empty((k, self.D)) if with_draws else None
        self.check(self.lib.kbo_forest_export(
            self._h, self._o, int(tree), *[out[a].ctypes.data for a in ("feature", "threshold", "left", "right", "value", "impurity",
                                                                         "n_node_samples", "weighted_n_node_samples")],
            draws.ctypes.data if draws is not None else None, k, None, None, self._stream()))
        out["counts"] = counts
        if draws is not None:
            out["draws"] = draws
        return out
