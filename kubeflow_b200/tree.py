"""What the tree surrogates on the GPU share (``ForestEngine``, ``GbrtEngine``): the fit of a history with its reuse, and the
candidate sweep through ``kbo_<kind>_fit`` / ``kbo_<kind>_sweep`` with skopt's EI / LCB / PI on the raw mean and standard
deviation.  A subclass gives its ``kbo_<kind>_create`` arguments, ``predict``, ``export`` and ``_fit(Xd, yd, N, D, counts)``: the
libkbo fit of the float32 / float64 CUDA tensors Xd (N × D) and yd, returning its status."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .gp import Best


class TreeEngine(L.Handle):
    _SWEEP_TAIL = ()               # arguments of kbo_<kind>_sweep between sigma_out and the stream

    def __init__(self, device: int, kind: str, create_args, acq: str, xi: float, kappa: float):
        self.acq, self.xi, self.kappa = acq, float(xi), float(kappa)
        super().__init__(device, kind, *create_args)
        self.N = self.D = 0
        self.y_opt = None
        self._hist = None          # (X, y) of the fitted model
        self.last_fit = None       # "fit" | "reuse"

    def _dev32(self, X) -> torch.Tensor:
        if isinstance(X, torch.Tensor):
            return X.to(device=f"cuda:{self.device}", dtype=torch.float32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(np.atleast_2d(X), dtype=np.float32)).to(f"cuda:{self.device}")

    def tell(self, X, y):
        """Fit the model to (X, y): X in the transformed space (cast to float32, as sklearn does), y raw and minimised.  The model
        is kept when X and y equal the last fit's."""
        self._tell(X, y)

    def _tell(self, X, y, counts=None):
        # counts: the forest's bootstrap counts, handed to _fit; a fit with them is never kept for reuse
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
        with torch.cuda.device(self.device):
            self.check(self._fit(Xd, yd, len(yh), Xh.shape[1], counts))
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
            self.check(getattr(self.lib, f"kbo_{self._kind}_sweep")(
                self._h, self._o, Xd.data_ptr(), int(M), int(global_offset), n, kinds, self.y_opt, self.xi, self.kappa,
                out.data_ptr() if n else None, mu.data_ptr() if mu is not None else None, sd.data_ptr() if sd is not None else None,
                *self._SWEEP_TAIL, self._stream()))
            raw = out.cpu().numpy()
        bests = [Best(float(raw[4 * i]), int(raw[4 * i + 1:4 * i + 2].view(np.int64)[0]), float(raw[4 * i + 2]), float(raw[4 * i + 3]))
                 for i in range(n)]
        return (bests, mu, sd) if return_arrays else bests

    def ask(self, Xc, global_offset: int = 0):
        """First-index argmax of the engine's acquisition over the candidates (transformed space)."""
        return self.sweep(Xc, [self.acq], global_offset)[0]

    def ask_multi(self, Xc, acqs, global_offset: int = 0):
        return self.sweep(Xc, list(acqs), global_offset)

    def last_timings(self) -> dict:
        return self._last_timings(("fit_ms", "sweep_ms"))
