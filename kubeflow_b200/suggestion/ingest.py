"""Request ingestion without the message tree (SURVEY.md §8(f)3).

Katib resends every finished trial, as strings, on every ``GetSuggestions`` call.  ``LazyRequest`` is what the gRPC server's
request deserializer returns instead of ``GetSuggestionsRequest.FromString(bytes)``: it keeps the wire bytes, parses only the
small ``experiment`` sub-message with protobuf, and lets the skopt service pull the trials through libkbo's scan
(``kbo_req_trials``, include/kbo.h) as NumPy arrays — names as 64-bit hashes, conditions, the objective, one double per
(trial, parameter).  Everything else (``request.trials`` for the services that walk the messages, error paths) falls back to
a full protobuf parse on first touch, so behaviour is the reference's; the scan only decides how fast the common case is.

Trials are recognised by the 64-bit FNV-1a hash of their name: two different names colliding (probability ~n²/2⁶⁵) would make
the later one look already told.

Mirrors kubeflow/katib pkg/suggestion/v1beta1/internal/trial.py ``Trial.convert`` (filter: succeeded trials carrying the
objective metric) and skopt/base_service.py ``getSuggestions`` (assignment lookup by parameter name, ``float``/``int``).
"""
from __future__ import annotations

import ctypes as C
import weakref
from dataclasses import dataclass

import numpy as np

from .. import _lib as L
from . import api_pb as api

MISSING = 0xFFFFFFFF


@dataclass
class TrialTable:
    """One row per trial of the request, in wire order."""
    n: int
    name_off: np.ndarray
    name_len: np.ndarray
    name_hash: np.ndarray        # uint64 FNV-1a of the name (kbo_hash64)
    condition: np.ndarray
    usable: np.ndarray           # bool: Trial.convert would keep it
    objective: np.ndarray        # float64, NaN unless objective_flags & 1
    objective_flags: np.ndarray
    objective_off: np.ndarray
    objective_len: np.ndarray
    values: np.ndarray           # (n, P) float64
    value_flags: np.ndarray      # (n, P) uint8: bit0 plain decimal literal, bit1 integer literal
    value_off: np.ndarray
    value_len: np.ndarray        # MISSING where the trial has no assignment of that name


def hash64(name: str) -> int:
    b = name.encode()
    return int(L.load().kbo_hash64(b, len(b)))


class LazyRequest:
    """Duck-types ``api.GetSuggestionsRequest`` for the servicers; adds ``trial_table`` for the fast path."""

    def __init__(self, data: bytes):
        self._data = bytes(data)
        self._msg = None
        self._exp = None
        self._h = C.c_void_p()
        self._lib = L.load()
        h = C.c_void_p()
        if self._lib.kbo_req_open(self._data, len(self._data), C.byref(h)) != L.KBO_OK:
            self._msg = api.GetSuggestionsRequest.FromString(self._data)    # malformed: let protobuf raise its own DecodeError
            return
        self._h = h
        weakref.finalize(self, self._lib.kbo_req_close, h)           # the scan's host buffers go with the request
        eo, el, cur, tot, nt = C.c_uint64(), C.c_uint64(), C.c_int32(), C.c_int32(), C.c_int32()
        self._lib.kbo_req_header(self._h, C.byref(eo), C.byref(el), C.byref(cur), C.byref(tot), C.byref(nt))
        self._exp_span = (eo.value, el.value)
        self.current_request_number, self.total_request_number, self.n_trials = cur.value, tot.value, nt.value

    @classmethod
    def FromString(cls, data: bytes) -> "LazyRequest":
        return cls(data)

    # -- protobuf view ------------------------------------------------------------------------------------------------
    @property
    def message(self):
        if self._msg is None:
            self._msg = api.GetSuggestionsRequest.FromString(self._data)
        return self._msg

    @property
    def experiment(self):
        if self._msg is not None:
            return self._msg.experiment
        if self._exp is None:
            o, n = self._exp_span
            self._exp = api.Experiment.FromString(self._data[o:o + n])
        return self._exp

    @property
    def trials(self):
        return self.message.trials

    def __getattr__(self, name):          # anything else (ByteSize, HasField, …) comes from the parsed message
        if name.startswith("_"):
            raise AttributeError(name)
        return getattr(self.message, name)

    @property
    def scanned(self) -> bool:
        return bool(self._h)

    # -- flat view ----------------------------------------------------------------------------------------------------
    def trial_table(self, param_names, select=None) -> TrialTable:
        """``select``: bool mask over the request's trials — only those rows get their assignments parsed."""
        if not self._h:
            raise RuntimeError("request bytes were not scannable")
        n, P = self.n_trials, len(param_names)
        names = (C.c_char_p * max(P, 1))(*[p.encode() for p in param_names])
        t = TrialTable(n, np.empty(n, np.uint64), np.empty(n, np.uint32), np.empty(n, np.uint64), np.empty(n, np.int32),
                       np.empty(n, np.uint8), np.empty(n, np.float64), np.empty(n, np.uint8), np.empty(n, np.uint64),
                       np.empty(n, np.uint32), np.empty((n, P), np.float64), np.empty((n, P), np.uint8),
                       np.empty((n, P), np.uint64), np.empty((n, P), np.uint32))
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
        mask = None if select is None else np.ascontiguousarray(select, dtype=np.uint8)
        if mask is not None and mask.shape != (n,):
            raise ValueError("select must have one entry per trial")
        sel = None if mask is None else ptr(mask)
        rc = self._lib.kbo_req_trials(self._h, P, names, ptr(t.name_off), ptr(t.name_len), ptr(t.name_hash), ptr(t.condition),
                                      ptr(t.usable), ptr(t.objective), ptr(t.objective_flags), ptr(t.objective_off),
                                      ptr(t.objective_len), ptr(t.values), ptr(t.value_flags), ptr(t.value_off), ptr(t.value_len), sel)
        if rc != L.KBO_OK:
            raise RuntimeError("malformed trial in request")
        t.usable = t.usable.astype(bool)
        return t

    def text(self, off: int, length: int) -> str:
        return self._data[int(off):int(off) + int(length)].decode()
