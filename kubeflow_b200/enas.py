"""The ENAS controller on the GPU (libkbo ``kbo_enas_*``) — the engine behind Katib's ``enas`` algorithm (the macro-search LSTM
controller of ENAS, trained by REINFORCE; FP64 restatement in oracle/enas_oracle.py): ``train()`` on a reward, ``sample()``
architectures."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L

PARAM_NAMES = ("w_lstm", "g_emb", "w_emb", "w_soft", "w_attn_1", "w_attn_2", "v_attn")
STAT_NAMES = ("nll", "ent", "kl", "loss", "baseline", "skip_rate")
DEFAULT_SETTINGS = dict(temperature=5.0, tanh_const=2.25, entropy_weight=1e-5, baseline_decay=0.999, learning_rate=5e-5,
                        skip_target=0.4, skip_weight=0.8)


def param_shapes(L_: int, H: int, n_ops: int) -> dict:
    """Shapes of the controller's parameters, in the order of the flat buffers."""
    return dict(w_lstm=(2 * H, 4 * H), g_emb=(1, H), w_emb=(n_ops, H), w_soft=(H, n_ops), w_attn_1=(H, H), w_attn_2=(H, H), v_attn=(H, 1))


def flatten(params: dict) -> np.ndarray:
    return np.concatenate([np.asarray(params[n], dtype=np.float32).ravel() for n in PARAM_NAMES])


def unflatten(flat: np.ndarray, L_: int, H: int, n_ops: int) -> dict:
    out, o = {}, 0
    for n, s in param_shapes(L_, H, n_ops).items():
        k = s[0] * s[1]
        out[n] = flat[o:o + k].reshape(s)
        o += k
    return out


class EnasController(L.Handle):
    """L layers, hidden size H, n_ops operations.  ``settings``: the keys of DEFAULT_SETTINGS; None for temperature,
    tanh_const, entropy_weight or skip_weight drops that term.  An arc is L(L+1)/2 integers: per layer its op, then one skip
    bit per earlier layer."""

    def __init__(self, num_layers: int, hidden: int, n_ops: int, settings: dict | None = None, seed: int = 0, device: int = 0):
        self.L, self.H, self.n_ops = int(num_layers), int(hidden), int(n_ops)
        self.A = self.L * (self.L + 1) // 2
        st = dict(DEFAULT_SETTINGS)
        st.update(settings or {})
        self.settings = st
        cs = L.KboEnasSettings(temperature=0.0 if st["temperature"] is None else float(st["temperature"]),
                               tanh_const=0.0 if st["tanh_const"] is None else float(st["tanh_const"]),
                               entropy_weight=0.0 if st["entropy_weight"] is None else float(st["entropy_weight"]),
                               baseline_decay=float(st["baseline_decay"]), learning_rate=float(st["learning_rate"]),
                               skip_target=float(st["skip_target"]), skip_weight=0.0 if st["skip_weight"] is None else float(st["skip_weight"]))
        super().__init__(device, "enas", self.L, self.H, self.n_ops, C.byref(cs), int(seed))
        self.n_par = sum(a * b for a, b in param_shapes(self.L, self.H, self.n_ops).values())

    def train(self, reward: float, steps: int, arcs=None) -> np.ndarray:
        """``steps`` REINFORCE steps on ``reward``; ``arcs`` (steps × L(L+1)/2) imposes the arcs.  Returns the per-step
        statistics (steps × 6: nll, ent, mean kl, loss, baseline, skip rate)."""
        steps = int(steps)
        dev = f"cuda:{self.device}"
        stats = torch.empty(max(steps, 1), len(STAT_NAMES), dtype=torch.float32, device=dev)
        ap = None
        if arcs is not None:
            a = torch.as_tensor(np.ascontiguousarray(np.asarray(arcs, dtype=np.int32).reshape(steps, self.A)), device=dev)
            ap = a.data_ptr()
        self.check(self.lib.kbo_enas_train(self._h, self._o, float(reward), steps, ap, stats.data_ptr(), self._stream()))
        return stats[:steps].cpu().numpy()

    def sample(self, k: int, uniforms=None, return_probs: bool = False):
        """k arcs (k × L(L+1)/2 int32 NumPy array).  ``uniforms`` (k × L(L+1)/2) imposes the draws.  ``return_probs``: also the
        op probabilities (k × L × n_ops) and P(skip = 1) per skip decision (k × L(L-1)/2), as NumPy arrays."""
        k = int(k)
        dev = f"cuda:{self.device}"
        arcs = torch.empty(k, self.A, dtype=torch.int32, device=dev)
        up = None
        if uniforms is not None:
            u = torch.as_tensor(np.ascontiguousarray(np.asarray(uniforms, dtype=np.float32).reshape(k, self.A)), device=dev)
            up = u.data_ptr()
        opp = torch.empty(k, self.L, self.n_ops, dtype=torch.float32, device=dev) if return_probs else None
        skp = torch.empty(k, max(self.L * (self.L - 1) // 2, 1), dtype=torch.float32, device=dev) if return_probs else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        self.check(self.lib.kbo_enas_sample(self._h, self._o, k, arcs.data_ptr(), up, ptr(opp), ptr(skp), self._stream()))
        out = arcs.cpu().numpy()
        if not return_probs:
            return out
        return out, opp.cpu().numpy(), skp[:, :self.L * (self.L - 1) // 2].cpu().numpy()

    def state(self) -> dict:
        """Parameters (dict of float32 arrays), Adam moments m and v (same layout), baseline, step and draw counter."""
        p, m, v = (np.empty(self.n_par, np.float32) for _ in range(3))
        b, t, d = C.c_float(), C.c_int64(), C.c_int64()
        self.check(self.lib.kbo_enas_state(self._h, self._o, p.ctypes.data, m.ctypes.data, v.ctypes.data, C.byref(b), C.byref(t),
                                           C.byref(d), self._stream()))
        u = lambda f: unflatten(f, self.L, self.H, self.n_ops)
        return dict(params=u(p), m=u(m), v=u(v), baseline=b.value, step=t.value, draws=d.value)

    def set_params(self, params: dict, m: dict | None = None, v: dict | None = None, baseline: float = 0.0, step: int = 0):
        """Replace the parameters (and optionally the moments; None: zero), the baseline and the Adam step count."""
        p = flatten(params)
        mm = flatten(m) if m is not None else None
        vv = flatten(v) if v is not None else None
        ptr = lambda a: a.ctypes.data if a is not None else None
        self.check(self.lib.kbo_enas_set_params(self._h, self._o, p.ctypes.data, ptr(mm), ptr(vv), float(baseline), int(step),
                                                self._stream()))

    def last_timings(self) -> dict:
        return self._last_timings(("train_ms", "sample_ms"))
