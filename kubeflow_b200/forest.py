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

from . import _lib as L
from .gp import Best

KINDS = {"RF": 0, "ET": 1}


class ForestEngine(L.Handle):
    def __init__(self, device: int = 0, *, kind: str = "RF", n_trees: int = 100, min_samples_leaf: int = 3, seed: int = 0,
                 acq: str = "ei", xi: float = 0.01, kappa: float = 1.96):
        if kind not in KINDS:
            raise ValueError(f"kind must be RF or ET, got {kind!r}")
        self.kind, self.n_trees = kind, int(n_trees)
        self.acq, self.xi, self.kappa = acq, float(xi), float(kappa)
        super().__init__(device, "forest", KINDS[kind], self.n_trees, int(min_samples_leaf), int(seed) & (2 ** 64 - 1))
        self.N = self.D = 0
        self.y_opt = None
        self._hist = None          # (X, y) of the fitted forest
        self.last_fit = None       # "fit" | "reuse"

    def _dev32(self, X) -> torch.Tensor:
        if isinstance(X, torch.Tensor):
            return X.to(device=f"cuda:{self.device}", dtype=torch.float32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(np.atleast_2d(X), dtype=np.float32)).to(f"cuda:{self.device}")

    def tell(self, X, y, counts=None):
        """Fit the forest to (X, y): X in the transformed space (cast to float32, as sklearn does), y minimised.  The forest is
        kept when X and y equal the last fit's.  ``counts``: optional T × N bootstrap counts (RF) replacing the drawn ones."""
        Xh = np.asarray(X, dtype=np.float64)
        Xh = Xh.reshape(len(Xh), -1)
        yh = np.asarray(y, dtype=np.float64).reshape(-1)
        if Xh.shape[0] != yh.shape[0]:
            raise ValueError("X and y must have the same number of rows")
        if counts is None and self._hist is not None and self._hist[0].shape == Xh.shape and np.array_equal(self._hist[0], Xh) \
                and np.array_equal(self._hist[1], yh):
            self.last_fit = "reuse"
            return
        self._hist = None
        Xd = self._dev32(Xh)
        yd = torch.from_numpy(np.ascontiguousarray(yh)).to(f"cuda:{self.device}")
        cd = None
        if counts is not None:
            cd = torch.from_numpy(np.ascontiguousarray(counts, dtype=np.int32).reshape(self.n_trees, len(yh))).to(f"cuda:{self.device}")
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_forest_fit(self._h, self._o, Xd.data_ptr(), yd.data_ptr(), len(yh), Xh.shape[1],
                                               cd.data_ptr() if cd is not None else None, self._stream()))
        self.N, self.D = Xh.shape
        self.y_opt = float(np.min(yh))
        self._hist = (Xh.copy(), yh.copy()) if counts is None else None
        self.last_fit = "fit"

    def _check(self, D):
        if self.N == 0:
            raise L.KboError(L.KBO_ERR_STATE, "ask() before tell(): call tell(X, y) first")
        if D != self.D:
            raise ValueError(f"candidates have D={D}, fit had D={self.D}")

    def sweep(self, Xc, acqs, global_offset: int = 0, return_arrays: bool = False):
        """One pass over the candidates for 0-3 acquisitions: a Best per acquisition (+ mu and sigma float64 CUDA tensors)."""
        Xd = self._dev32(Xc)
        M, D = Xd.shape
        self._check(D)
        for a in acqs:
            if a not in L.ACQS:
                raise ValueError(f"acq must be one of {sorted(L.ACQS)}, got {a!r}")
        n = len(acqs)
        kinds = (C.c_int32 * max(n, 1))(*[L.ACQS[a] for a in acqs])
        dev = f"cuda:{self.device}"
        out = torch.empty(4 * max(n, 1), dtype=torch.float64, device=dev)
        mu = torch.empty(M, dtype=torch.float64, device=dev) if return_arrays else None
        sd = torch.empty(M, dtype=torch.float64, device=dev) if return_arrays else None
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_forest_sweep(self._h, self._o, Xd.data_ptr(), int(M), int(global_offset), n, kinds, self.y_opt,
                                                 self.xi, self.kappa, out.data_ptr() if n else None,
                                                 mu.data_ptr() if mu is not None else None,
                                                 sd.data_ptr() if sd is not None else None, self._stream()))
            raw = out.cpu().numpy()
        bests = [Best(float(raw[4 * i]), int(raw[4 * i + 1:4 * i + 2].view(np.int64)[0]), float(raw[4 * i + 2]), float(raw[4 * i + 3]))
                 for i in range(n)]
        return (bests, mu, sd) if return_arrays else bests

    def ask(self, Xc, global_offset: int = 0):
        """First-index argmax of the engine's acquisition over the candidates (transformed space)."""
        return self.sweep(Xc, [self.acq], global_offset)[0]

    def ask_multi(self, Xc, acqs, global_offset: int = 0):
        return self.sweep(Xc, list(acqs), global_offset)

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

    def last_timings(self) -> dict:
        return self._last_timings(("fit_ms", "sweep_ms"))
