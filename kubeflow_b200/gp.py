"""Host-side GP engine: fixed-θ tell (fit) / ask (sweep + argmax) on one H100 through libkbo's C ABI.

Mirrors what Katib's skopt service does per request at fixed θ (SURVEY.md §3.1):
``skopt.Optimizer.tell`` -> ``GaussianProcessRegressor.fit`` ($SK/_gpr.py:233-368) and
``_gaussian_acquisition`` over a sampled candidate set -> ``X_cand[np.argmin(values)]``.
PyTorch is used for device storage and stream handles only; all arithmetic is in libkbo.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib as L


@dataclass
class Best:
    value: float   # acquisition value to maximise (EI, PI, or -(mu - kappa*sigma) for LCB)
    index: int     # global candidate index, lowest index among equal maxima
    mu: float      # posterior mean at that candidate (raw y scale)
    std: float     # posterior std at that candidate (raw y scale)


class GPEngine(L.Handle):
    def __init__(self, device: int = 0, *, kernel: str = "matern52", length_scale=1.0, amplitude: float = 1.0,
                 noise: float = 1e-10, acq: str = "ei", xi: float = 0.01, kappa: float = 1.96,
                 normalize_y: bool = True, var_mode: str = "auto", tc_k_span: int = 0, scratch_limit: int | None = None,
                 tc_fast: bool | None = None, rank_tc: bool | None = None, rank_prefix: int | None = None,
                 lazy_inverse: bool | None = None):
        if kernel not in L.KERNELS:
            raise ValueError(f"kernel must be one of {sorted(L.KERNELS)}, got {kernel!r}")
        if acq not in L.ACQS:
            raise ValueError(f"acq must be one of {sorted(L.ACQS)}, got {acq!r}")
        if var_mode not in L.VAR_MODES:
            raise ValueError(f"var_mode must be one of {sorted(L.VAR_MODES)}, got {var_mode!r}")
        super().__init__(device)
        self.kernel, self.acq, self.var_mode = kernel, acq, var_mode
        self.length_scale = np.atleast_1d(np.asarray(length_scale, dtype=np.float64)).copy()
        self.amplitude, self.noise, self.xi, self.kappa = float(amplitude), float(noise), float(xi), float(kappa)
        self.normalize_y, self.tc_k_span = bool(normalize_y), int(tc_k_span)
        self.N = self.D = 0
        self.scratch_limit = 4 << 30 if scratch_limit is None else int(scratch_limit)   # libkbo's default
        if scratch_limit is not None:
            self.check(self.lib.kbo_set_scratch_limit(self._h, int(scratch_limit)))
        if tc_fast is not None:
            self.check(self.lib.kbo_set_tc_fast(self._h, int(bool(tc_fast))))
        if rank_tc is not None:
            self.check(self.lib.kbo_set_rank_tc(self._h, int(bool(rank_tc))))
        if lazy_inverse is not None:
            self.check(self.lib.kbo_set_lazy_inverse(self._h, int(bool(lazy_inverse))))
        if rank_prefix is not None:
            self.check(self.lib.kbo_set_rank_prefix(self._h, int(rank_prefix)))
        self._best_dev = torch.empty(4, dtype=torch.float64, device=f"cuda:{self.device}")

    # -- plumbing ----------------------------------------------------------------------------------
    def _params(self):
        self._ls_arr = (C.c_double * len(self.length_scale))(*self.length_scale)
        return L.KboParams(kernel=L.KERNELS[self.kernel], acq=L.ACQS[self.acq], normalize_y=int(self.normalize_y),
                           var_mode=L.VAR_MODES[self.var_mode], amplitude=self.amplitude, noise=self.noise, xi=self.xi,
                           kappa=self.kappa, length_scale=self._ls_arr, n_length_scale=len(self.length_scale),
                           tc_k_span=self.tc_k_span)

    @staticmethod
    def _as_host_f64(a):
        return np.ascontiguousarray(np.asarray(a, dtype=np.float64))

    # -- tell --------------------------------------------------------------------------------------
    def tell(self, X, y):
        """Fit at fixed θ.  X: (N, D), y: (N,) — NumPy (copied H2D inside) or float64 CUDA tensors."""
        p = self._params()
        if isinstance(X, torch.Tensor):
            if not (X.is_cuda and y.is_cuda and X.dtype == torch.float64 and y.dtype == torch.float64):
                raise ValueError("tensor inputs must be float64 CUDA tensors")
            X, y = X.contiguous(), y.contiguous().reshape(-1)
            self._keep = (X, y)
            N, D = X.shape
            xp, yp, on_host = X.data_ptr(), y.data_ptr(), 0
        else:
            X, y = self._as_host_f64(X), self._as_host_f64(y).reshape(-1)
            if X.ndim != 2 or X.shape[0] != y.shape[0]:
                raise ValueError(f"X must be (N, D) and y (N,), got {X.shape} and {y.shape}")
            self._keep = (X, y)
            N, D = X.shape
            xp, yp, on_host = X.ctypes.data, y.ctypes.data, 1
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_fit(self._h, xp, yp, int(N), int(D), C.byref(p), on_host, self._stream())
        self.check(rc)
        self.N, self.D = int(N), int(D)
        return self

    def room(self) -> int:
        """How many more trials `append` can add in place (0: `tell` the whole history again)."""
        return int(self.lib.kbo_fit_room(self._h))

    def append(self, x, y: float):
        """One more trial at the fitted θ: bordered Cholesky row instead of a refit (kbo_fit_append; what skopt's constant-liar
        `ask(n_points=k)` needs k-1 times per request, and what a steady Katib experiment needs once per finished trial)."""
        if self.N == 0:
            raise L.KboError(L.KBO_ERR_STATE, "append() before tell(): call tell(X, y) first")
        x = self._as_host_f64(x).reshape(-1)
        if x.shape[0] != self.D:
            raise ValueError(f"x has {x.shape[0]} values, fit had D={self.D}")
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_fit_append(self._h, x.ctypes.data, float(y), 1, self._stream())
        self.check(rc)
        self.N += 1
        return self

    def rebase(self, n_keep: int, y=None):
        """Keep the first `n_keep` trials (optionally with new targets): drops constant-liar rows, swaps a lie for the
        observed value — no refactorisation (kbo_fit_rebase)."""
        yp = None
        if y is not None:
            y = self._as_host_f64(y).reshape(-1)
            if y.shape[0] < n_keep:
                raise ValueError(f"y has {y.shape[0]} values, need n_keep={n_keep}")
            yp = y.ctypes.data
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_fit_rebase(self._h, int(n_keep), yp, 1, self._stream())
        self.check(rc)
        self.N = int(n_keep)
        return self

    def fit_info(self):
        lml, ym, ys, yo, info = C.c_double(), C.c_double(), C.c_double(), C.c_double(), C.c_int32()
        rc = self.lib.kbo_fit_info(self._h, C.byref(lml), C.byref(ym), C.byref(ys), C.byref(yo), C.byref(info), self._stream())
        self.check(rc)
        return dict(lml=lml.value, y_mean=ym.value, y_std=ys.value, y_opt=yo.value, info=info.value)

    def last_contenders(self) -> int:
        """How many candidates the last tensor-core sweep re-evaluated in FP64."""
        return int(self.lib.kbo_last_contenders(self._h))

    def last_rank_error(self) -> float:
        """Largest |σ²(1 product) − σ²(3 products)| on the calibration rows of the last one-product sweep (kbo_set_tc_fast)."""
        return float(self.lib.kbo_last_rank_error(self._h))

    def last_rank_mu_error(self) -> float:
        """Largest |mean(ranking pass) − mean(FP64 K* kernel)| on the calibration rows of the last ranking sweep (normalised y)."""
        return float(self.lib.kbo_last_rank_mu_error(self._h))

    def last_prefix_survivors(self) -> int:
        """Candidates the last pruning pass kept (kbo_set_rank_prefix); -1 if it did not run."""
        return int(self.lib.kbo_last_prefix_survivors(self._h))

    def last_unrefined(self) -> int:
        """0: the last tensor-core suggestion was decided in FP64 among every candidate that could be the maximum;
        1: among the best 4096 by fp32 value (window overflow); 2: not refined (exact ties beyond the cap, or a grid of 2^31 or
        more rows)."""
        return int(self.lib.kbo_last_unrefined(self._h))

    def fp64_peak_tflops(self) -> float:
        """Test / bench hook: the FP64 tensor-core (DMMA) rate of this GPU, measured on register-resident operands."""
        out = C.c_double(0.0)
        self.check(self.lib.kbo_debug_fp64_peak(self._h, C.byref(out)))
        return float(out.value)

    def rank_pass(self, Xc, mode: int, want_plane: bool = False):
        """Test hook: the ranking pass alone (mode 0: FP64 K* + one-product cluster kernel, 1: tensor-core K* + wgmma
        kernel) -> normalised mean, normalised variance (float32 CUDA tensors) and optionally the fp16 K* hi plane."""
        dev = f"cuda:{self.device}"
        if not isinstance(Xc, torch.Tensor):
            Xc = torch.as_tensor(np.ascontiguousarray(Xc), device=dev)
        Xc = Xc.contiguous()
        dt = L.KBO_F64 if Xc.dtype == torch.float64 else L.KBO_F32
        M = Xc.shape[0]
        npad = (self.N + 255) // 256 * 256
        mu = torch.empty(M, dtype=torch.float32, device=dev)
        var = torch.empty(M, dtype=torch.float32, device=dev)
        plane = torch.empty((M, npad), dtype=torch.float16, device=dev) if want_plane else None
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_debug_rank_pass(self._h, Xc.data_ptr(), dt, int(M), int(mode), mu.data_ptr(), var.data_ptr(),
                                              plane.data_ptr() if want_plane else None, self._stream())
            self.check(rc)
            torch.cuda.current_stream(self.device).synchronize()
        return mu, var, plane

    def kstar_pass(self, Xc, store_cols: int = -1, plane=None):
        """Test hook: the tensor-core K* kernel alone -> (normalised mean of the M candidates, fp16 K* plane of rows_pad × Npad,
        rows_pad = M rounded up to 256).  With store_cols >= 0 only the 128-column tiles covering the first store_cols columns are
        written; pass ``plane`` to see what the kernel leaves alone."""
        dev = f"cuda:{self.device}"
        if not isinstance(Xc, torch.Tensor):
            Xc = torch.as_tensor(np.ascontiguousarray(Xc), device=dev)
        Xc = Xc.contiguous()
        dt = L.KBO_F64 if Xc.dtype == torch.float64 else L.KBO_F32
        M = Xc.shape[0]
        rows_pad, npad = (M + 255) // 256 * 256, (self.N + 255) // 256 * 256
        mu = torch.empty(rows_pad, dtype=torch.float32, device=dev)
        if plane is None:
            plane = torch.empty((rows_pad, npad), dtype=torch.float16, device=dev)
        assert plane.shape == (rows_pad, npad) and plane.dtype == torch.float16 and plane.is_contiguous()
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_debug_kstar(self._h, Xc.data_ptr(), dt, int(M), int(store_cols), mu.data_ptr(), plane.data_ptr(), self._stream())
            self.check(rc)
            torch.cuda.current_stream(self.device).synchronize()
        return mu[:M], plane

    def rank_rows(self, Xc, tile_pairs: int = -1, slice_rows: int = 131072):
        """Test hook: the normalised mean and variance the pruning pass (``tile_pairs`` >= 1: the variance over the first
        tile_pairs pairs of 256-trial tiles, an upper bound) or the full ranking pass (-1) computes for every row of the CUDA
        tensor ``Xc``, as float32 CUDA tensors.  The grid goes through in slices of ``slice_rows`` (the hook's scratch is
        slice_rows × N fp16)."""
        if not (isinstance(Xc, torch.Tensor) and Xc.is_cuda):
            raise ValueError("rank_rows takes a CUDA tensor")
        Xc = Xc.contiguous()
        dt = L.KBO_F64 if Xc.dtype == torch.float64 else L.KBO_F32
        M = Xc.shape[0]
        mu = torch.empty(M, dtype=torch.float32, device=Xc.device)
        var = torch.empty(M, dtype=torch.float32, device=Xc.device)
        with torch.cuda.device(self.device):
            for r0 in range(0, M, slice_rows):
                m = min(slice_rows, M - r0)
                rc = self.lib.kbo_debug_rank_rows(self._h, Xc[r0:].data_ptr(), dt, int(m), int(tile_pairs), mu[r0:].data_ptr(),
                                                  var[r0:].data_ptr(), self._stream())
                self.check(rc)
            torch.cuda.current_stream(self.device).synchronize()
        return mu, var

    STAGES = ("lazy-prune", "prune", "prune-interval", "interval", "window")

    def record_stages(self, on: bool = True):
        """Test hook: keep, for every stage of each later ask / ask_multi and every acquisition, the bounds it pruned with and
        its survivors (``stages()``).  Recording reads them back; it changes no arithmetic."""
        self.check(self.lib.kbo_debug_record_stages(self._h, int(bool(on))))
        return self

    def stages(self):
        """The stages the last ask / ask_multi ran, in order: dicts of stage, acq, cal_n, n (survivors counted), E, E_mu,
        dvar_raw / dmu_raw (the maxima E and E_mu came from), lb (lower bound on the maximum; NaN: none), thr (the survivor
        threshold), delta (the three-product window) and survivors (grid-local indices, at most the stage's cap)."""
        out = []
        acq_names = {v: k for k, v in L.ACQS.items()}
        for i in range(int(self.lib.kbo_debug_stage_count(self._h))):
            ints, fl = (C.c_int32 * 4)(), (C.c_float * 7)()
            n = self.lib.kbo_debug_stage(self._h, i, ints, fl, None, 0)
            self.check(min(n, 0))
            lst = np.empty(max(n, 1), dtype=np.int32)
            self.lib.kbo_debug_stage(self._h, i, ints, fl, lst.ctypes.data, n)
            out.append(dict(stage=self.STAGES[ints[0]], acq=acq_names[ints[1]], cal_n=int(ints[2]), n=int(ints[3]),
                            **dict(zip(("E", "E_mu", "dvar_raw", "dmu_raw", "lb", "thr", "delta"), (float(v) for v in fl))),
                            survivors=np.sort(lst[:n].astype(np.int64))))
        return out

    def lml_grad(self):
        """(lml, grad) of the last tell; grad w.r.t. (log amplitude, log noise, log ℓ_1..ℓ_P) as a NumPy array."""
        info = self.fit_info()
        g = np.empty(2 + len(self.length_scale), dtype=np.float64)
        rc = self.lib.kbo_lml_grad(self._h, g.ctypes.data_as(C.POINTER(C.c_double)), len(g), self._stream())
        self.check(rc)
        return info["lml"], g

    def _theta_params(self, thetas):
        """KboParams array for a list of θ dicts (length_scale / noise / amplitude; the engine's own values where absent), and
        the length-scale buffers it points to."""
        arr = (L.KboParams * len(thetas))()
        keep = []
        for g, th in enumerate(thetas):
            ls = np.atleast_1d(np.asarray(th.get("length_scale", self.length_scale), dtype=np.float64))
            buf = (C.c_double * len(ls))(*ls)
            keep.append(buf)
            arr[g] = L.KboParams(kernel=L.KERNELS[self.kernel], acq=L.ACQS[self.acq], normalize_y=int(self.normalize_y),
                                 var_mode=L.VAR_MODES[self.var_mode], amplitude=float(th.get("amplitude", self.amplitude)),
                                 noise=float(th.get("noise", self.noise)), xi=self.xi, kappa=self.kappa, length_scale=buf,
                                 n_length_scale=len(ls), tc_k_span=self.tc_k_span)
        return arr, keep

    def lml_batch(self, X, y, thetas, return_info: bool = False):
        """Log-marginal likelihood of several θ over one history in one call (kbo_lml_batch: the factorisations run concurrently).
        ``thetas``: list of dicts with any of length_scale / noise / amplitude (the engine's own values where absent).
        Returns a float64 NumPy array, −inf where the Gram matrix is not positive definite (with ``return_info``, also each θ's
        1-based failed pivot, 0 if none).  The fitted state is untouched."""
        X, y = self._as_host_f64(X), self._as_host_f64(y).reshape(-1)
        N, D = X.shape
        G = len(thetas)
        arr, keep = self._theta_params(thetas)
        out = np.empty(G, dtype=np.float64)
        info = (C.c_int32 * G)()
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_lml_batch(self._h, X.ctypes.data, y.ctypes.data, int(N), int(D), int(G), arr, 1,
                                        out.ctypes.data_as(C.POINTER(C.c_double)), info, self._stream())
        self.check(rc)
        return (out, np.array(info[:], dtype=np.int32)) if return_info else out

    def lml_grad_batch(self, X, y, thetas, return_info: bool = False):
        """Log-marginal likelihood and its gradient for several θ over one history in one call (kbo_lml_grad_batch: each θ on
        its own stream, results independent of the batch).  ``thetas`` as for ``lml_batch``; every θ needs the same number of
        length scales P.  Returns (lml[G], grad[G, 2 + P]) as float64 NumPy arrays, grad in ``lml_grad``'s order (log amplitude,
        log noise, log ℓ_1..ℓ_P); a θ whose Gram matrix is not positive definite has lml −inf and a zero gradient (with
        ``return_info``, also each θ's 1-based failed pivot, 0 if none).  The fitted state is untouched."""
        X, y = self._as_host_f64(X), self._as_host_f64(y).reshape(-1)
        N, D = X.shape
        G = len(thetas)
        arr, keep = self._theta_params(thetas)
        P = arr[0].n_length_scale if G else 1
        lml = np.empty(G, dtype=np.float64)
        grad = np.empty((G, 2 + P), dtype=np.float64)
        info = (C.c_int32 * max(G, 1))()
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_lml_grad_batch(self._h, X.ctypes.data, y.ctypes.data, int(N), int(D), int(G), arr, 1,
                                             lml.ctypes.data_as(C.POINTER(C.c_double)), grad.ctypes.data_as(C.POINTER(C.c_double)),
                                             info, self._stream())
        self.check(rc)
        return (lml, grad, np.array(info[:G], dtype=np.int32)) if return_info else (lml, grad)

    @staticmethod
    def lml_grad_lane_bytes(N: int, D: int, P: int) -> int:
        """Device memory one θ of ``lml_grad_batch`` takes (kbo_i_lml_grad_lane_bytes in fit.cu); a batch needs G times this
        within the engine's scratch limit."""
        ld, nb = (N + 63) // 64 * 64, (N + 63) // 64
        return 8 * (3 * ld * ld + 2 * ld * D + 3 * ld + nb * nb * (2 + P) + (2 + P) + 64 * 64 + 512 + 16) + 4 * 4

    def state(self):
        """Copies of L (lower), W = L^-1 and alpha as float64 CUDA tensors (parity tests)."""
        N, dev = self.N, f"cuda:{self.device}"
        Lm = torch.empty(N, N, dtype=torch.float64, device=dev)
        Wm = torch.empty(N, N, dtype=torch.float64, device=dev)
        al = torch.empty(N, dtype=torch.float64, device=dev)
        rc = self.lib.kbo_fit_state(self._h, Lm.data_ptr(), Wm.data_ptr(), al.data_ptr(), self._stream())
        self.check(rc)
        torch.cuda.current_stream(self.device).synchronize()
        return Lm, Wm, al

    # -- multi-GPU exchange through the C ABI (kbo_comm_*, kbo_allreduce_argmax) --------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        """The 128-byte NCCL unique id (call on one rank, hand the bytes to every rank's ``comm_init``)."""
        buf = C.create_string_buffer(128)
        rc = L.load().kbo_comm_unique_id(buf)
        if rc != L.KBO_OK:
            raise L.KboError(rc, "kbo_comm_unique_id failed (libnccl.so.2 not loadable?)")
        return buf.raw

    def comm_init(self, n_ranks: int, rank: int, unique_id: bytes):
        """Collective over the ranks' engines: afterwards ``ask(..., allreduce=True)`` returns the global argmax."""
        if len(unique_id) != 128:
            raise ValueError("unique_id must be the 128 bytes of comm_unique_id()")
        with torch.cuda.device(self.device):
            self.check(self.lib.kbo_comm_init(self._h, int(n_ranks), int(rank), C.c_char_p(unique_id)))
        return self

    def comm_size(self) -> int:
        return int(self.lib.kbo_comm_size(self._h))

    # -- ask ---------------------------------------------------------------------------------------
    def ask(self, Xc, global_offset: int = 0, return_arrays: bool = False, allreduce: bool = False):
        """Sweep the candidate grid; returns Best (and mu/std/acq float64 CUDA tensors if asked).  ``allreduce``: combine the
        ranks' results into the global first-index argmax inside libkbo (kbo_allreduce_argmax; needs ``comm_init``)."""
        dev = f"cuda:{self.device}"
        ptr, on_host, dt, M, D, Xc = self._rows(Xc)
        if self.N == 0:
            raise L.KboError(L.KBO_ERR_STATE, "ask() before tell(): call tell(X, y) first")
        if D != self.D:
            raise ValueError(f"candidates have D={D}, fit had D={self.D}")
        mu = std = acq = None
        mp = sp = ap = None
        if return_arrays:
            mu = torch.empty(M, dtype=torch.float64, device=dev)
            std = torch.empty(M, dtype=torch.float64, device=dev)
            acq = torch.empty(M, dtype=torch.float64, device=dev)
            mp, sp, ap = mu.data_ptr(), std.data_ptr(), acq.data_ptr()
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_sweep(self._h, ptr, dt, int(M), int(global_offset), on_host, mp, sp, ap,
                                    self._best_dev.data_ptr(), self._stream())
            self.check(rc)
            if allreduce:
                self.check(self.lib.kbo_allreduce_argmax(self._h, self._best_dev.data_ptr(), self._stream()))
            b = L.KboBest()
            rc = self.lib.kbo_best_to_host(self._h, self._best_dev.data_ptr(), C.byref(b), self._stream())
            self.check(rc)
        best = Best(b.value, int(b.index), b.mu, b.std)
        return (best, mu, std, acq) if return_arrays else best

    def _rows(self, X):
        """(pointer, on_host, dtype code, rows, keep-alive) of a candidate / point matrix: NumPy or a CUDA tensor."""
        if isinstance(X, torch.Tensor):
            if not X.is_cuda or X.dtype not in (torch.float64, torch.float32):
                raise ValueError("candidate tensor must be a float64/float32 CUDA tensor")
            X = X.contiguous()
            M, D = X.shape
            return X.data_ptr(), 0, L.KBO_F64 if X.dtype == torch.float64 else L.KBO_F32, M, D, X
        X = np.ascontiguousarray(X)
        if X.dtype not in (np.float64, np.float32):
            X = X.astype(np.float64)
        M, D = X.shape
        return X.ctypes.data, 1, L.KBO_F64 if X.dtype == np.float64 else L.KBO_F32, M, D, X

    def ask_multi(self, Xc, acqs, global_offset: int = 0):
        """Sweep the candidate grid once for several acquisitions (kbo_sweep_multi): one Best per entry of ``acqs`` (1-3
        distinct names of "ei", "lcb", "pi"), each what ``ask`` with that acquisition returns on the same fit and grid."""
        ptr, on_host, dt, M, D, keep = self._rows(Xc)
        if self.N == 0:
            raise L.KboError(L.KBO_ERR_STATE, "ask_multi() before tell(): call tell(X, y) first")
        if D != self.D:
            raise ValueError(f"candidates have D={D}, fit had D={self.D}")
        for a in acqs:
            if a not in L.ACQS:
                raise ValueError(f"acq must be one of {sorted(L.ACQS)}, got {a!r}")
        n = len(acqs)
        kinds = (C.c_int32 * max(n, 1))(*[L.ACQS[a] for a in acqs])
        out = torch.empty(4 * max(n, 1), dtype=torch.float64, device=f"cuda:{self.device}")
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_sweep_multi(self._h, ptr, dt, int(M), int(global_offset), on_host, int(n), kinds, out.data_ptr(), self._stream())
            self.check(rc)
            bests = []
            for i in range(n):
                b = L.KboBest()
                self.check(self.lib.kbo_best_to_host(self._h, out.data_ptr() + 32 * i, C.byref(b), self._stream()))
                bests.append(Best(b.value, int(b.index), b.mu, b.std))
        del keep
        return bests

    def last_decisions(self):
        """Per acquisition of the last ask / ask_multi: (unrefined, contenders, prefix survivors) as kbo_last_unrefined,
        kbo_last_contenders and kbo_last_prefix_survivors report them for a single sweep."""
        u, c, p = (C.c_int32 * 3)(), (C.c_int32 * 3)(), (C.c_int32 * 3)()
        n = self.lib.kbo_last_decisions(self._h, 3, u, c, p)
        if n < 0:
            self.check(n)
        return [(int(u[i]), int(c[i]), int(p[i])) for i in range(n)]

    def predict_mean(self, X) -> np.ndarray:
        """FP64 posterior mean (raw y scale) at the rows of X (kbo_predict_mean; does not form a lazy fit's inverse)."""
        ptr, on_host, dt, n, D, keep = self._rows(np.atleast_2d(X) if not isinstance(X, torch.Tensor) else X)
        if self.N == 0:
            raise L.KboError(L.KBO_ERR_STATE, "predict_mean() before tell(): call tell(X, y) first")
        if D != self.D:
            raise ValueError(f"points have D={D}, fit had D={self.D}")
        mu = np.empty(n, dtype=np.float64)
        with torch.cuda.device(self.device):
            rc = self.lib.kbo_predict_mean(self._h, ptr, dt, int(n), on_host, mu.ctypes.data, self._stream())
        self.check(rc)
        del keep
        return mu

    # -- one call, host buffers (the end-to-end entry bench.py times) -------------------------------
    def suggest_host(self, X, y, Xc, global_offset: int = 0):
        X, y = self._as_host_f64(X), self._as_host_f64(y).reshape(-1)
        Xc = np.ascontiguousarray(Xc)
        if Xc.dtype not in (np.float64, np.float32):
            Xc = Xc.astype(np.float64)
        dt = L.KBO_F64 if Xc.dtype == np.float64 else L.KBO_F32
        p = self._params()
        b, t = L.KboBest(), L.KboTimings()
        rc = self.lib.kbo_suggest_host(self._h, X.ctypes.data, y.ctypes.data, X.shape[0], X.shape[1], Xc.ctypes.data, dt,
                                       Xc.shape[0], int(global_offset), C.byref(p), C.byref(b), C.byref(t))
        self.check(rc)
        self.N, self.D = X.shape
        return Best(b.value, int(b.index), b.mu, b.std), t.as_dict()

    # -- standalone HBM-bound acquisition pass (fp32 mu_n / var_n, 8 B per candidate) ------------------
    def acq_argmax_f32(self, mu_n: torch.Tensor, var_n: torch.Tensor, *, y_mean: float, y_std: float, y_opt: float,
                       global_offset: int = 0, acq_out: torch.Tensor | None = None) -> Best:
        rc = self.lib.kbo_acq_argmax(self._h, mu_n.data_ptr(), var_n.data_ptr(), mu_n.numel(), int(global_offset),
                                     L.ACQS[self.acq], y_mean, y_std, y_opt, self.xi, self.kappa,
                                     acq_out.data_ptr() if acq_out is not None else None, self._best_dev.data_ptr(),
                                     self._stream())
        self.check(rc)
        torch.cuda.current_stream(self.device).synchronize()
        v = self._best_dev.cpu()
        return Best(float(v[0]), int(v[1:2].view(torch.int64)[0]), float(v[2]), float(v[3]))
