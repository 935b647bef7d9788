"""CMA-ES sampler on the GPU (libkbo ``kbo_cma_*``) — host-side mirror of goptuna's ``cmaes`` sampler that Katib's
``cmaes`` algorithm uses (SURVEY.md §8(a) A9): ``ask()`` a population, ``tell()`` its fitness.  ``SepCmaEs``
(``kbo_sepcma_*``) is the separable variant with a diagonal C, for spaces of up to 4096 parameters."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L


class _Strategy(L.Handle):
    """What the full and the separable sampler share: ``kbo_<kind>_create``, ask, tell, stop_flags and restart."""
    kind = ""

    def __init__(self, mean, sigma: float, popsize: int | None = None, seed: int = 0, device: int = 0):
        mean = np.ascontiguousarray(np.asarray(mean, dtype=np.float64))
        self.D = int(mean.shape[0])
        self.popsize = int(popsize) if popsize else 4 + int(3 * np.log(self.D))
        super().__init__(device, self.kind, self.D, self.popsize, mean.ctypes.data_as(C.POINTER(C.c_double)), float(sigma), int(seed))
        self._X = torch.empty(self.popsize, self.D, dtype=torch.float64, device=f"cuda:{self.device}")

    def _fn(self, name):
        return getattr(self.lib, f"kbo_{self.kind}_{name}")

    def ask(self, z: torch.Tensor | None = None) -> torch.Tensor:
        """Population (popsize × D float64 CUDA tensor).  ``z``: optional popsize×D standard normals (CUDA float64)."""
        zp = None
        if z is not None:
            if not (z.is_cuda and z.dtype == torch.float64 and tuple(z.shape) == (self.popsize, self.D)):
                raise ValueError("z must be a float64 CUDA tensor of shape (popsize, D)")
            z = z.contiguous()
            zp = z.data_ptr()
        self.check(self._fn("ask")(self._h, self._o, self._X.data_ptr(), zp, self._stream()))
        return self._X

    def tell(self, fitness):
        f = fitness if isinstance(fitness, torch.Tensor) else torch.tensor(np.asarray(fitness, dtype=np.float64))
        f = f.to(device=f"cuda:{self.device}", dtype=torch.float64).contiguous()
        if f.numel() != self.popsize:
            raise ValueError(f"fitness must have {self.popsize} entries")
        self.check(self._fn("tell")(self._h, self._o, f.data_ptr(), self._stream()))

    def stop_flags(self):
        """(flags, funhist, term) of the termination test run at the end of the last tell: the bit mask (TOLFUN=1, TOLX=2,
        TOLXUP=4, NOEFFECTCOORD=8, NOEFFECTAXIS=16 (full CMA-ES only), CONDITIONCOV=32; 0 before a run's first tell), the
        history ring of each generation's best and worst fitness (2·term values) and term."""
        flags, term = C.c_uint32(), C.c_int32()
        hist = np.zeros(2 * (10 + -(-30 * self.D // 4)))     # room for the largest ring (λ = 4)
        self.check(self._fn("stop_flags")(self._h, self._o, C.byref(flags), hist.ctypes.data, C.byref(term),
                                          self._stream()))
        return flags.value, hist[:2 * term.value].copy(), term.value

    def restart(self, popsize: int, mean, sigma: float):
        """Start a new run in place (IPOP / BIPOP): population `popsize`, C = I, zero paths, strategy generation 0.  The
        built-in sampler's stream continues, so no earlier draw repeats."""
        mean = np.ascontiguousarray(np.asarray(mean, dtype=np.float64))
        if mean.shape != (self.D,):
            raise ValueError(f"mean must have {self.D} entries")
        self.check(self._fn("restart")(self._h, self._o, int(popsize), mean.ctypes.data_as(C.POINTER(C.c_double)),
                                       float(sigma)))
        if int(popsize) != self.popsize:
            self.popsize = int(popsize)
            self._X = torch.empty(self.popsize, self.D, dtype=torch.float64, device=f"cuda:{self.device}")


class CmaEs(_Strategy):
    """Full CMA-ES (D <= 128): C is D×D with its eigenbasis B."""
    kind = "cma"

    def state(self, with_Y: bool = False) -> dict:
        D, lam = self.D, self.popsize
        out = dict(mean=np.empty(D), sigma=np.empty(1), C=np.empty((D, D)), p_sigma=np.empty(D), pc=np.empty(D), B=np.empty((D, D)),
                   d=np.empty(D))
        Y = np.empty((lam, D)) if with_Y else None
        gen = C.c_int64()
        ptr = lambda a: a.ctypes.data if a is not None else None
        self.check(self.lib.kbo_cma_state(self._h, self._o, ptr(out["mean"]), ptr(out["sigma"]), ptr(out["C"]),
                                          ptr(out["p_sigma"]), ptr(out["pc"]), ptr(out["B"]), ptr(out["d"]), ptr(Y),
                                          C.byref(gen), self._stream()))
        out["sigma"] = float(out["sigma"][0])
        out["generation"] = gen.value
        if with_Y:
            out["Y"] = Y
        return out

    def set_margin(self, dims: dict, alpha: float | None = None):
        """CMA-ES with Margin on the discrete dimensions ``dims``: {index: sorted cube levels (1-D array, 2 or more) or an
        arithmetic range (first, step, count)}.  ``alpha`` is the margin (default 1/(D·λ), recomputed at restarts).  From
        the next ask on, samples carry each discrete coordinate encoded to its level, and A starts at ones.  An empty
        ``dims`` turns the margin off.  Not between an ask and its tell."""
        idx = sorted(int(i) for i in dims)
        offs, lev, arith = [0], [], []
        for i in idx:
            v = dims[i]
            if isinstance(v, tuple):
                arith += [float(v[0]), float(v[1]), float(v[2])]
            else:
                lev.append(np.asarray(v, dtype=np.float64).ravel())
                arith += [0.0, 0.0, 0.0]
            offs.append(offs[-1] + (0 if isinstance(v, tuple) else len(lev[-1])))
        d = np.array(idx, dtype=np.int32)
        o = np.array(offs, dtype=np.int64)
        lv = np.ascontiguousarray(np.concatenate(lev) if lev else np.zeros(1))
        ar = np.array(arith if arith else [0.0], dtype=np.float64)
        self.check(self.lib.kbo_cma_set_margin(self._h, self._o, len(idx), d.ctypes.data, o.ctypes.data, lv.ctypes.data,
                                               ar.ctypes.data, float(alpha or 0.0)))
        self.margin_dims = idx

    def margin_state(self) -> dict:
        """A, the mean after the last tell's update and before its margin correction, and α (needs set_margin)."""
        A, mb, alpha = np.empty(self.D), np.empty(self.D), C.c_double()
        self.check(self.lib.kbo_cma_margin_state(self._h, self._o, A.ctypes.data, mb.ctypes.data, C.byref(alpha),
                                                 self._stream()))
        return dict(A=A, mean_before=mb, alpha=alpha.value)

    def set_lr_adapt(self, on: bool):
        """Learning-rate adaptation (LRA-CMA-ES, Optuna's ``CmaEsSampler(lr_adapt=True)``) on or off; either way the
        adaptation's state starts afresh (E = V = 0, η = 1), as it does at every restart.  Not between an ask and its
        tell, and not with a margin set."""
        self.check(self.lib.kbo_cma_set_lr_adapt(self._h, self._o, 1 if on else 0))

    def lr_state(self) -> dict:
        """The adaptation's state after the last tell: E_mean (D), E_Sigma (D×D), V_mean, V_Sigma, eta_mean, eta_Sigma
        (needs set_lr_adapt(True))."""
        Em, ES, V, eta = np.empty(self.D), np.empty((self.D, self.D)), np.empty(2), np.empty(2)
        self.check(self.lib.kbo_cma_lra_state(self._h, self._o, Em.ctypes.data, ES.ctypes.data, V.ctypes.data, eta.ctypes.data,
                                              self._stream()))
        return dict(E_mean=Em, E_Sigma=ES, V_mean=float(V[0]), V_Sigma=float(V[1]), eta_mean=float(eta[0]), eta_Sigma=float(eta[1]))

    def run_synthetic(self, fitness: str, generations: int):
        """BASELINE config 4: `generations` full generations on the device with a built-in fitness."""
        kind = {"sphere": 0, "rastrigin": 1}[fitness]
        best, ms, sw = C.c_double(), C.c_float(), C.c_double()
        self.check(self.lib.kbo_cma_run_synthetic(self._h, self._o, kind, int(generations), C.byref(best), C.byref(ms),
                                                  C.byref(sw)))
        return dict(best_f=best.value, elapsed_ms=ms.value, generations_per_s=generations / (ms.value * 1e-3), jacobi_sweeps=sw.value)


class SepCmaEs(_Strategy):
    """Separable CMA-ES (libkbo ``kbo_sepcma_*``, D <= 4096; ``oracle/sepcma_oracle.py``): C is diagonal, so there is no
    basis, and ``state()`` returns C as its diagonal (D,) and d = √C."""
    kind = "sepcma"

    def state(self, with_Y: bool = False) -> dict:
        D, lam = self.D, self.popsize
        out = dict(mean=np.empty(D), sigma=np.empty(1), C=np.empty(D), p_sigma=np.empty(D), pc=np.empty(D), d=np.empty(D))
        Y = np.empty((lam, D)) if with_Y else None
        gen = C.c_int64()
        ptr = lambda a: a.ctypes.data if a is not None else None
        self.check(self.lib.kbo_sepcma_state(self._h, self._o, ptr(out["mean"]), ptr(out["sigma"]), ptr(out["C"]),
                                             ptr(out["p_sigma"]), ptr(out["pc"]), ptr(out["d"]), ptr(Y), C.byref(gen),
                                             self._stream()))
        out["sigma"] = float(out["sigma"][0])
        out["generation"] = gen.value
        if with_Y:
            out["Y"] = Y
        return out
