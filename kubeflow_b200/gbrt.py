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

from . import _lib as L
from .gp import Best

SKOPT_QUANTILES = (0.16, 0.5, 0.84)


class GbrtEngine(L.Handle):
    def __init__(self, device: int = 0, *, quantiles=SKOPT_QUANTILES, n_estimators: int = 30, acq: str = "ei", xi: float = 0.01,
                 kappa: float = 1.96):
        q = tuple(float(v) for v in quantiles)
        if len(q) != 3:
            raise ValueError(f"quantiles must hold three values (lower, middle, upper), got {quantiles!r}")
        self.quantiles, self.n_estimators = q, int(n_estimators)
        self.acq, self.xi, self.kappa = acq, float(xi), float(kappa)
        super().__init__(device, "gbrt", (C.c_double * 3)(*q), self.n_estimators)
        self.N = self.D = 0
        self.y_opt = None
        self._hist = None          # (X, y) of the fitted model
        self.last_fit = None       # "fit" | "reuse"

    def _dev32(self, X) -> torch.Tensor:
        if isinstance(X, torch.Tensor):
            return X.to(device=f"cuda:{self.device}", dtype=torch.float32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(np.atleast_2d(X), dtype=np.float32)).to(f"cuda:{self.device}")

    def tell(self, X, y):
        """Fit the three chains to (X, y): X in the transformed space (cast to float32, as sklearn does), y raw and minimised.  The
        model is kept when X and y equal the last fit's."""
        Xh = np.asarray(X, dtype=np.float64)
        Xh = Xh.reshape(len(Xh), -1)
        yh = np.asarray(y, dtype=np.float64).reshape(-1)
        if Xh.shape[0] != yh.shape[0]:
            raise ValueError("X and y must have the same number of rows")
        if self._hist is not None and self._hist[0].shape == Xh.shape and np.array_equal(self._hist[0], Xh) \
                and np.array_equal(self._hist[1], yh):
            self.last_fit = "reuse"
            return
        self._hist = None
        Xd = self._dev32(Xh)
        yd = torch.from_numpy(np.ascontiguousarray(yh)).to(f"cuda:{self.device}")
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_gbrt_fit(self._h, self._o, Xd.data_ptr(), yd.data_ptr(), len(yh), Xh.shape[1], self._stream()))
        self.N, self.D = Xh.shape
        self.y_opt = float(np.min(yh))
        self._hist = (Xh.copy(), yh.copy())
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
            self.check(self.lib.kbo_gbrt_sweep(self._h, self._o, Xd.data_ptr(), int(M), int(global_offset), n, kinds, self.y_opt,
                                               self.xi, self.kappa, out.data_ptr() if n else None,
                                               mu.data_ptr() if mu is not None else None,
                                               sd.data_ptr() if sd is not None else None, None, self._stream()))
            raw = out.cpu().numpy()
        bests = [Best(float(raw[4 * i]), int(raw[4 * i + 1:4 * i + 2].view(np.int64)[0]), float(raw[4 * i + 2]), float(raw[4 * i + 3]))
                 for i in range(n)]
        return (bests, mu, sd) if return_arrays else bests

    def ask(self, Xc, global_offset: int = 0):
        """First-index argmax of the engine's acquisition over the candidates (transformed space)."""
        return self.sweep(Xc, [self.acq], global_offset)[0]

    def ask_multi(self, Xc, acqs, global_offset: int = 0):
        return self.sweep(Xc, list(acqs), global_offset)

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

    def last_timings(self) -> dict:
        return self._last_timings(("fit_ms", "sweep_ms"))
