"""ctypes binding of include/kbo.h.  There is no CPU path: a missing libkbo.so or a missing CUDA device
raises; nothing here falls back to NumPy."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libkbo.so")

KBO_OK, KBO_ERR_INVALID, KBO_ERR_CUDA, KBO_ERR_NOT_PD, KBO_ERR_NOMEM, KBO_ERR_STATE = 0, -1, -2, -3, -4, -5
KERNELS = {"rbf": 0, "matern52": 1}
ACQS = {"ei": 0, "lcb": 1, "pi": 2}
VAR_MODES = {"f64": 0, "tc": 1, "auto": 2}
KBO_F64, KBO_F32 = 0, 1


class KboParams(C.Structure):
    _fields_ = [("kernel", C.c_int32), ("acq", C.c_int32), ("normalize_y", C.c_int32), ("var_mode", C.c_int32),
                ("amplitude", C.c_double), ("noise", C.c_double), ("xi", C.c_double), ("kappa", C.c_double),
                ("length_scale", C.POINTER(C.c_double)), ("n_length_scale", C.c_int32), ("tc_k_span", C.c_int32)]


class KboBest(C.Structure):
    _fields_ = [("value", C.c_double), ("index", C.c_int64), ("mu", C.c_double), ("std", C.c_double)]


class KboTimings(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("fit_ms", C.c_float), ("sweep_ms", C.c_float), ("d2h_ms", C.c_float),
                ("total_ms", C.c_float), ("var_kernel_ms", C.c_float), ("cross_kernel_ms", C.c_float),
                ("acq_kernel_ms", C.c_float), ("launches", C.c_int32), ("chunks", C.c_int32), ("calib_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class KboError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libkbo error {code}: {msg}")
        self.code = code


class KboInvalidArgument(KboError, ValueError):
    """KBO_ERR_INVALID — the gRPC layer maps this to INVALID_ARGUMENT."""


class KboNotPositiveDefinite(KboError):
    """KBO_ERR_NOT_PD — same condition sklearn reports as LinAlgError in GPR.fit ($SK/_gpr.py:353-362)."""


# every symbol include/kbo.h declares (tests/test_abi.py checks the .so exports exactly these)
EXPORTS = ["kbo_version", "kbo_create", "kbo_destroy", "kbo_last_error", "kbo_set_scratch_limit", "kbo_last_contenders", "kbo_set_tc_fast", "kbo_last_rank_error", "kbo_set_rank_tc", "kbo_last_rank_mu_error", "kbo_last_unrefined", "kbo_set_rank_prefix", "kbo_last_prefix_survivors", "kbo_set_lazy_inverse", "kbo_fit", "kbo_fit_append", "kbo_fit_room", "kbo_fit_rebase",
           "kbo_fit_info", "kbo_lml_grad", "kbo_lml_batch", "kbo_lml_grad_batch", "kbo_fit_state", "kbo_sweep", "kbo_sweep_multi", "kbo_last_decisions", "kbo_predict_mean", "kbo_best_to_host",
           "kbo_comm_unique_id", "kbo_comm_init", "kbo_comm_destroy", "kbo_comm_size", "kbo_allreduce_argmax", "kbo_suggest_host", "kbo_last_timings",
           "kbo_gram", "kbo_potrf", "kbo_trtri", "kbo_acq_argmax",
           "kbo_req_open", "kbo_req_close", "kbo_req_header", "kbo_req_trials", "kbo_hash64",
           "kbo_cma_create", "kbo_cma_destroy", "kbo_cma_ask", "kbo_cma_tell", "kbo_cma_state", "kbo_cma_run_synthetic",
           "kbo_cma_stop_flags", "kbo_cma_restart", "kbo_cma_set_margin", "kbo_cma_margin_state", "kbo_cma_set_lr_adapt",
           "kbo_cma_lra_state",
           "kbo_sepcma_create", "kbo_sepcma_destroy", "kbo_sepcma_ask", "kbo_sepcma_tell", "kbo_sepcma_state", "kbo_sepcma_stop_flags",
           "kbo_sepcma_restart",
           "kbo_tpe_create", "kbo_tpe_destroy", "kbo_tpe_tell", "kbo_tpe_ask", "kbo_tpe_state", "kbo_tpe_last_survivors", "kbo_tpe_last_timings",
           "kbo_tpe_ask_shard", "kbo_tpe_pick",
           "kbo_mvtpe_create", "kbo_mvtpe_destroy", "kbo_mvtpe_tell", "kbo_mvtpe_ask", "kbo_mvtpe_state", "kbo_mvtpe_last_survivors",
           "kbo_mvtpe_last_timings", "kbo_mvtpe_ask_shard", "kbo_mvtpe_pick",
           "kbo_forest_create", "kbo_forest_destroy", "kbo_forest_fit", "kbo_forest_sweep", "kbo_forest_predict", "kbo_forest_export",
           "kbo_forest_last_timings",
           "kbo_gbrt_create", "kbo_gbrt_destroy", "kbo_gbrt_fit", "kbo_gbrt_sweep", "kbo_gbrt_predict", "kbo_gbrt_export",
           "kbo_gbrt_last_timings",
           "kbo_enas_create", "kbo_enas_destroy", "kbo_enas_train", "kbo_enas_sample", "kbo_enas_state", "kbo_enas_set_params",
           "kbo_enas_last_timings"]


class KboEnasSettings(C.Structure):
    _fields_ = [("temperature", C.c_double), ("tanh_const", C.c_double), ("entropy_weight", C.c_double), ("baseline_decay", C.c_double),
                ("learning_rate", C.c_double), ("skip_target", C.c_double), ("skip_weight", C.c_double)]


_lib = None


def load() -> C.CDLL:
    """dlopen libkbo.so (built in-tree by kubeflow_b200/build.py) and declare the prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        # a fresh checkout has no built library (it is git-ignored): build it in-tree if nvcc is here, else fail loudly
        import shutil
        if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
            from . import build as _build
            _build.build()
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing and could not be built: run `python -c 'import __graft_entry__ as g; "
                              "g.build()'` (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    pd = C.POINTER(C.c_double)
    lib.kbo_version.restype = C.c_int
    lib.kbo_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.kbo_destroy.argtypes = [vp]
    lib.kbo_destroy.restype = None
    lib.kbo_last_error.argtypes = [vp]
    lib.kbo_last_error.restype = C.c_char_p
    lib.kbo_set_scratch_limit.argtypes = [vp, C.c_uint64]
    lib.kbo_fit_append.argtypes = [vp, vp, C.c_double, C.c_int, vp]
    lib.kbo_fit_room.argtypes = [vp]
    lib.kbo_req_open.argtypes = [vp, C.c_uint64, C.POINTER(vp)]
    lib.kbo_req_close.argtypes = [vp]
    lib.kbo_req_close.restype = None
    lib.kbo_req_header.argtypes = [vp] + [vp] * 5
    lib.kbo_req_trials.argtypes = [vp, C.c_int32, C.POINTER(C.c_char_p)] + [vp] * 14
    lib.kbo_hash64.argtypes = [vp, C.c_uint64]
    lib.kbo_hash64.restype = C.c_uint64
    lib.kbo_fit_rebase.argtypes = [vp, C.c_int32, vp, C.c_int, vp]
    lib.kbo_last_contenders.argtypes = [vp]
    lib.kbo_set_tc_fast.argtypes = [vp, C.c_int]
    lib.kbo_last_rank_error.argtypes = [vp]
    lib.kbo_last_rank_error.restype = C.c_double
    lib.kbo_set_rank_tc.argtypes = [vp, C.c_int]
    lib.kbo_last_rank_mu_error.argtypes = [vp]
    lib.kbo_last_rank_mu_error.restype = C.c_double
    lib.kbo_last_unrefined.argtypes = [vp]
    lib.kbo_set_rank_prefix.argtypes = [vp, C.c_int]
    lib.kbo_last_prefix_survivors.argtypes = [vp]
    lib.kbo_set_lazy_inverse.argtypes = [vp, C.c_int]
    lib.kbo_comm_unique_id.argtypes = [vp]
    lib.kbo_comm_init.argtypes = [vp, i32, i32, vp]
    lib.kbo_comm_destroy.argtypes = [vp]
    lib.kbo_comm_size.argtypes = [vp]
    lib.kbo_allreduce_argmax.argtypes = [vp, vp, vp]
    lib.kbo_debug_rank_pass.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp, vp]
    lib.kbo_debug_kstar.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp]
    lib.kbo_debug_rank_rows.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp]
    lib.kbo_debug_record_stages.argtypes = [vp, i32]
    lib.kbo_debug_stage_count.argtypes = [vp]
    lib.kbo_debug_stage.argtypes = [vp, i32, vp, vp, vp, i32]
    lib.kbo_debug_fit_stream_path.argtypes = [vp, i32]
    lib.kbo_debug_fit_graph.argtypes = [vp, vp]
    lib.kbo_debug_forest_sweep.argtypes = [vp, vp, vp]
    lib.kbo_debug_fp64_peak.argtypes = [vp, pd]
    lib.kbo_debug_dgemm_sm90.argtypes = [vp, i32, i32, i32, i32, vp, i32, vp, i32, vp, i32, dbl, dbl, i32, i32, i32, vp]
    lib.kbo_fit.argtypes = [vp, vp, vp, i32, i32, C.POINTER(KboParams), C.c_int, vp]
    lib.kbo_fit_info.argtypes = [vp, pd, pd, pd, pd, C.POINTER(i32), vp]
    lib.kbo_fit_state.argtypes = [vp, vp, vp, vp, vp]
    lib.kbo_lml_grad.argtypes = [vp, pd, i32, vp]
    lib.kbo_lml_batch.argtypes = [vp, vp, vp, i32, i32, i32, C.POINTER(KboParams), C.c_int, pd, C.POINTER(i32), vp]
    lib.kbo_lml_grad_batch.argtypes = [vp, vp, vp, i32, i32, i32, C.POINTER(KboParams), C.c_int, pd, pd, C.POINTER(i32), vp]
    lib.kbo_sweep.argtypes = [vp, vp, i32, i64, i64, C.c_int, vp, vp, vp, vp, vp]
    lib.kbo_sweep_multi.argtypes = [vp, vp, i32, i64, i64, C.c_int, i32, vp, vp, vp]
    lib.kbo_last_decisions.argtypes = [vp, i32, vp, vp, vp]
    lib.kbo_predict_mean.argtypes = [vp, vp, i32, i32, C.c_int, vp, vp]
    lib.kbo_best_to_host.argtypes = [vp, vp, C.POINTER(KboBest), vp]
    lib.kbo_suggest_host.argtypes = [vp, vp, vp, i32, i32, vp, i32, i64, i64, C.POINTER(KboParams), C.POINTER(KboBest),
                                     C.POINTER(KboTimings)]
    lib.kbo_last_timings.argtypes = [vp, C.POINTER(KboTimings)]
    lib.kbo_gram.argtypes = [vp, vp, i32, i32, i32, dbl, dbl, vp, i32, vp]
    lib.kbo_potrf.argtypes = [vp, vp, i32, i32, vp, vp]
    lib.kbo_trtri.argtypes = [vp, vp, i32, i32, vp, i32, vp]
    lib.kbo_acq_argmax.argtypes = [vp, vp, vp, i64, i64, i32, dbl, dbl, dbl, dbl, dbl, vp, vp, vp]
    lib.kbo_cma_create.argtypes = [vp, C.POINTER(vp), i32, i32, pd, dbl, C.c_uint64]
    lib.kbo_cma_destroy.argtypes = [vp]
    lib.kbo_cma_destroy.restype = None
    lib.kbo_cma_ask.argtypes = [vp, vp, vp, vp, vp]
    lib.kbo_cma_tell.argtypes = [vp, vp, vp, vp]
    lib.kbo_cma_state.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(i64), vp]
    lib.kbo_cma_run_synthetic.argtypes = [vp, vp, i32, i32, pd, C.POINTER(C.c_float), pd]
    lib.kbo_cma_stop_flags.argtypes = [vp, vp, C.POINTER(C.c_uint32), vp, C.POINTER(i32), vp]
    lib.kbo_cma_restart.argtypes = [vp, vp, i32, pd, dbl]
    lib.kbo_cma_set_margin.argtypes = [vp, vp, i32, vp, vp, vp, vp, dbl]
    lib.kbo_cma_margin_state.argtypes = [vp, vp, vp, vp, pd, vp]
    lib.kbo_cma_set_lr_adapt.argtypes = [vp, vp, i32]
    lib.kbo_cma_lra_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.kbo_sepcma_create.argtypes = [vp, C.POINTER(vp), i32, i32, pd, dbl, C.c_uint64]
    lib.kbo_sepcma_destroy.argtypes = [vp]
    lib.kbo_sepcma_destroy.restype = None
    lib.kbo_sepcma_ask.argtypes = [vp, vp, vp, vp, vp]
    lib.kbo_sepcma_tell.argtypes = [vp, vp, vp, vp]
    lib.kbo_sepcma_state.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(i64), vp]
    lib.kbo_sepcma_stop_flags.argtypes = [vp, vp, C.POINTER(C.c_uint32), vp, C.POINTER(i32), vp]
    lib.kbo_sepcma_restart.argtypes = [vp, vp, i32, pd, dbl]
    lib.kbo_tpe_create.argtypes = [vp, C.POINTER(vp), i32, vp, vp, vp, vp, vp, dbl, dbl, C.c_uint64]
    lib.kbo_tpe_destroy.argtypes = [vp]
    lib.kbo_tpe_destroy.restype = None
    lib.kbo_tpe_tell.argtypes = [vp, vp, vp, vp, i32, C.c_int, vp]
    lib.kbo_tpe_ask.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.kbo_tpe_state.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp]
    lib.kbo_tpe_last_survivors.argtypes = [vp, vp, vp, i32]
    lib.kbo_tpe_last_timings.argtypes = [vp, vp, vp, i32]
    lib.kbo_tpe_ask_shard.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp]
    lib.kbo_tpe_pick.argtypes = [vp, vp, i32, vp, vp, vp]
    lib.kbo_mvtpe_create.argtypes = [vp, C.POINTER(vp), i32, vp, vp, vp, vp, vp, C.c_uint64]
    lib.kbo_mvtpe_destroy.argtypes = [vp]
    lib.kbo_mvtpe_destroy.restype = None
    lib.kbo_mvtpe_tell.argtypes = [vp, vp, vp, vp, i32, C.c_int, vp]
    lib.kbo_mvtpe_ask.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.kbo_mvtpe_state.argtypes = [vp, vp, i32, vp, vp, vp, vp, i32, vp, vp, vp]
    lib.kbo_mvtpe_last_survivors.argtypes = [vp, vp, vp, i32]
    lib.kbo_mvtpe_last_timings.argtypes = [vp, vp, vp, i32]
    lib.kbo_mvtpe_ask_shard.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp]
    lib.kbo_mvtpe_pick.argtypes = [vp, vp, i32, vp, vp, vp]
    lib.kbo_forest_create.argtypes = [vp, C.POINTER(vp), i32, i32, i32, C.c_uint64]
    lib.kbo_forest_destroy.argtypes = [vp]
    lib.kbo_forest_destroy.restype = None
    lib.kbo_forest_fit.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.kbo_forest_sweep.argtypes = [vp, vp, vp, i64, i64, i32, vp, dbl, dbl, dbl, vp, vp, vp, vp]
    lib.kbo_forest_predict.argtypes = [vp, vp, vp, i32, C.c_int, vp, vp, vp]
    lib.kbo_forest_export.argtypes = [vp, vp, i32] + [vp] * 9 + [i32, vp, vp, vp]
    lib.kbo_forest_last_timings.argtypes = [vp, vp, vp, i32]
    lib.kbo_gbrt_create.argtypes = [vp, C.POINTER(vp), vp, i32]
    lib.kbo_gbrt_destroy.argtypes = [vp]
    lib.kbo_gbrt_destroy.restype = None
    lib.kbo_gbrt_fit.argtypes = [vp, vp, vp, vp, i32, i32, vp]
    lib.kbo_gbrt_sweep.argtypes = [vp, vp, vp, i64, i64, i32, vp, dbl, dbl, dbl, vp, vp, vp, vp, vp]
    lib.kbo_gbrt_predict.argtypes = [vp, vp, vp, i32, C.c_int, vp, vp, vp, vp]
    lib.kbo_gbrt_export.argtypes = [vp, vp, i32, i32] + [vp] * 7 + [i32, vp, vp, vp]
    lib.kbo_gbrt_last_timings.argtypes = [vp, vp, vp, i32]
    lib.kbo_enas_create.argtypes = [vp, C.POINTER(vp), i32, i32, i32, C.POINTER(KboEnasSettings), C.c_uint64]
    lib.kbo_enas_destroy.argtypes = [vp]
    lib.kbo_enas_destroy.restype = None
    lib.kbo_enas_train.argtypes = [vp, vp, dbl, i32, vp, vp, vp]
    lib.kbo_enas_sample.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    lib.kbo_enas_state.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.kbo_enas_set_params.argtypes = [vp, vp, vp, vp, vp, C.c_float, i64, vp]
    lib.kbo_enas_last_timings.argtypes = [vp, vp, vp, i32]
    lib.kbo_tc_variance_raw.argtypes = [vp, vp, vp, i64, vp, vp, i32, vp, dbl, vp, vp, i32, vp]
    for name in EXPORTS + ["kbo_tc_variance_raw", "kbo_debug_rank_pass", "kbo_debug_kstar", "kbo_debug_rank_rows", "kbo_debug_record_stages",
                           "kbo_debug_stage_count", "kbo_debug_stage", "kbo_debug_fp64_peak", "kbo_debug_dgemm_sm90",
                           "kbo_debug_fit_stream_path", "kbo_debug_fit_graph", "kbo_debug_forest_sweep"]:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("kbo_version",):
            fn.restype = C.c_int
    _lib = lib
    return lib


def check(lib, handle, code: int):
    if code == KBO_OK:
        return
    msg = lib.kbo_last_error(handle).decode() if handle else "no handle"
    if code == KBO_ERR_INVALID:
        raise KboInvalidArgument(code, msg)
    if code == KBO_ERR_NOT_PD:
        raise KboNotPositiveDefinite(code, msg)
    raise KboError(code, msg)


class Handle:
    """Owner of one libkbo handle (``kbo_create`` on ``device``) and, given ``kind``, of one engine object made on it by
    ``kbo_<kind>_create(handle, &object, *create_args)``.  ``close()`` destroys the object, then the handle; it is idempotent
    and safe after an ``__init__`` that failed partway (a failed ``kbo_<kind>_create`` closes the handle before raising)."""

    def __init__(self, device: int = 0, kind: str | None = None, *create_args):
        if not torch.cuda.is_available():
            raise RuntimeError("kubeflow_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.lib = load()
        self.device = int(device)
        h = C.c_void_p()
        rc = self.lib.kbo_create(C.byref(h), self.device)
        if rc != KBO_OK:
            raise KboError(rc, "kbo_create failed (no usable CUDA device?)")
        self._h = h
        if kind is not None:
            self._kind, o = kind, C.c_void_p()
            try:
                self.check(getattr(self.lib, f"kbo_{kind}_create")(self._h, C.byref(o), *create_args))
            except BaseException:
                self.close()
                raise
            self._o = o

    def close(self):
        if getattr(self, "_o", None):
            getattr(self.lib, f"kbo_{self._kind}_destroy")(self._o)
            self._o = C.c_void_p()
        if getattr(self, "_h", None):
            self.lib.kbo_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, code: int):
        check(self.lib, self._h, code)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _last_survivors(self) -> np.ndarray:
        """``kbo_<kind>_last_survivors``: the count (NULL buffer), then the int32 entries."""
        fn = getattr(self.lib, f"kbo_{self._kind}_last_survivors")
        n = fn(self._h, self._o, None, 0)
        out = np.zeros(max(n, 0), np.int32)
        if n > 0:
            fn(self._h, self._o, out.ctypes.data, n)
        return out

    def _last_timings(self, names) -> dict:
        """``kbo_<kind>_last_timings``: one float32 millisecond figure per name."""
        ms = np.zeros(len(names), np.float32)
        getattr(self.lib, f"kbo_{self._kind}_last_timings")(self._h, self._o, ms.ctypes.data, len(names))
        return dict(zip(names, ms.tolist()))
