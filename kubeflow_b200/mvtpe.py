"""Multivariate TPE on the GPU (libkbo ``kbo_mvtpe_*``) — the engine behind Katib's ``multivariate-tpe`` algorithm (Optuna's
``TPESampler(multivariate=True)`` on a flat space; FP64 restatement in oracle/mvtpe_oracle.py): ``tell()`` trials, ``ask()``
points."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L

FLOAT, INT, CAT = 0, 1, 2


class MvTpe(L.Handle):
    """params: list of ``("float", lo, hi)``, ``("int", lo, hi, step)`` or ``("cat", n_categories)``.  Values are in parameter
    units: integers are grid points lo + j·step <= hi, categoricals are observed and suggested as category indices."""

    def __init__(self, params, seed: int = 0, device: int = 0):
        self.params = [tuple(p) for p in params]
        self.D = len(self.params)
        kinds = np.zeros(self.D, np.int32)
        lo, hi, q = np.zeros(self.D), np.ones(self.D), np.ones(self.D)
        levels = np.zeros(self.D, np.int32)
        for d, p in enumerate(self.params):
            if p[0] == "float":
                kinds[d], lo[d], hi[d] = FLOAT, p[1], p[2]
            elif p[0] == "int":
                kinds[d], lo[d], hi[d], q[d] = INT, p[1], p[2], p[3]
            elif p[0] == "cat":
                kinds[d], levels[d] = CAT, p[1]
            else:
                raise ValueError(f"unknown parameter kind {p[0]!r}")
        self.kinds = kinds
        super().__init__(device, "mvtpe", self.D, kinds.ctypes.data, lo.ctypes.data, hi.ctypes.data, q.ctypes.data, levels.ctypes.data,
                         int(seed))
        self.n = 0

    def tell(self, X, losses):
        """Append trials in told order: X (n × D, parameter units) and their losses (minimised; NaN is refused)."""
        X = np.ascontiguousarray(np.asarray(X, dtype=np.float64).reshape(-1, self.D))
        y = np.ascontiguousarray(np.asarray(losses, dtype=np.float64).reshape(-1))
        if X.shape[0] != y.shape[0]:
            raise ValueError("X and losses must have the same number of rows")
        if X.shape[0]:
            self.check(self.lib.kbo_mvtpe_tell(self._h, self._o, X.ctypes.data, y.ctypes.data, X.shape[0], 1, self._stream()))
            self.n += X.shape[0]

    def ask(self, k: int = 1, n_candidates: int = 24, candidates: torch.Tensor | None = None, return_details: bool = False,
            shard: bool = False):
        """k suggestions (k × D float64 NumPy array).  ``candidates``: optional k × D × n_candidates float64 CUDA tensor.
        ``return_details``: also the winning indices, the candidates as scored (CUDA tensor, integers on their grid) and the
        FP32 scores with their bounds (k × n_candidates × 2 CUDA tensor).  ``shard``: when the default process group has more
        than one rank, every rank draws and scores its ``shard_rows`` block of the candidates and one exchange gives all ranks
        the suggestions a one-GPU ask would make (``dist.sharded_ask``); every rank must then make the same calls."""
        k, M = int(k), int(n_candidates)
        if shard:
            if candidates is not None or return_details:
                raise ValueError("candidates and return_details cannot be combined with shard")
            import torch.distributed as dist
            if dist.is_initialized() and dist.get_world_size() > 1:
                from .dist import sharded_ask
                cdev = torch.device("cuda", self.device) if dist.get_backend() == "nccl" else torch.device("cpu")
                return sharded_ask(lambda lo, hi: self.ask_shard(k, M, lo, hi), lambda idx: self.pick(k, idx), M, k, cdev)
        dev = f"cuda:{self.device}"
        cp = None
        if candidates is not None:
            if not (candidates.is_cuda and candidates.dtype == torch.float64 and tuple(candidates.shape) == (k, self.D, M)):
                raise ValueError("candidates must be a float64 CUDA tensor of shape (k, D, n_candidates)")
            candidates = candidates.contiguous()
            cp = candidates.data_ptr()
        x = torch.empty(k, self.D, dtype=torch.float64, device=dev)
        idx = torch.empty(k, dtype=torch.int64, device=dev) if return_details else None
        cout = torch.empty(k, self.D, M, dtype=torch.float64, device=dev) if return_details else None
        sc = torch.empty(k, M, 2, dtype=torch.float32, device=dev) if return_details else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        self.check(self.lib.kbo_mvtpe_ask(self._h, self._o, k, M, cp, x.data_ptr(), ptr(idx), ptr(cout), ptr(sc), self._stream()))
        out = x.cpu().numpy()
        if not return_details:
            return out
        return dict(x=out, index=idx.cpu().numpy(), candidates=cout, scores=sc, survivors=self.last_survivors())

    def state(self) -> dict:
        """{"below": ..., "above": ..., "n_below"}; each group is dict(w, sigma, mu, cat_rows): the weights of its observations
        in told order followed by the prior's, sigma per parameter (NaN for categoricals), the observations' values (m × D) and,
        per categorical, an observation row's entry at its own category and elsewhere (NaN for other kinds)."""
        out = {}
        for g, name in ((0, "below"), (1, "above")):
            m, nb = C.c_int32(), C.c_int32()
            self.check(self.lib.kbo_mvtpe_state(self._h, self._o, g, None, None, None, None, 0, C.byref(m), C.byref(nb), self._stream()))
            w, sg, mu, cr = np.empty(m.value + 1), np.empty(self.D), np.empty((m.value, self.D)), np.empty((self.D, 2))
            self.check(self.lib.kbo_mvtpe_state(self._h, self._o, g, w.ctypes.data, sg.ctypes.data, mu.ctypes.data, cr.ctypes.data,
                                                m.value + 1, None, None, self._stream()))
            out[name] = dict(w=w, sigma=sg, mu=mu, cat_rows=cr)
            out["n_below"] = nb.value
        return out

    def ask_shard(self, k: int, n_candidates: int, lo: int, hi: int):
        """One shard of a sharded ask: candidates [lo, hi) of n_candidates, drawn by their global index.  Returns this shard's
        winner per point as (FP64 values, global indices) NumPy arrays; an empty shard (lo == hi) gives (-inf, n_candidates).
        The ask counter advances as one ``ask`` advances it."""
        dev = f"cuda:{self.device}"
        val = torch.empty((int(k),), dtype=torch.float64, device=dev)
        idx = torch.empty((int(k),), dtype=torch.int64, device=dev)
        self.check(self.lib.kbo_mvtpe_ask_shard(self._h, self._o, int(k), int(n_candidates), int(lo), int(hi), None, val.data_ptr(),
                                                idx.data_ptr(), self._stream()))
        return val.cpu().numpy(), idx.cpu().numpy()

    def pick(self, k: int, index) -> np.ndarray:
        """The suggestions (k × D) at the winning global indices ``index`` (one per point) of the last shard ask,
        regenerated from their draws: what ``ask`` returns when those candidates win."""
        dev = f"cuda:{self.device}"
        idx = torch.as_tensor(np.asarray(index, dtype=np.int64).reshape((int(k),))).to(dev)
        x = torch.empty(int(k), self.D, dtype=torch.float64, device=dev)
        self.check(self.lib.kbo_mvtpe_pick(self._h, self._o, int(k), idx.data_ptr(), x.data_ptr(), self._stream()))
        return x.cpu().numpy()

    def last_survivors(self) -> np.ndarray:
        return self._last_survivors()

    def last_timings(self) -> dict:
        return self._last_timings(("models_and_draws_ms", "score_fp32_ms", "decide_fp64_ms", "final_ms"))
