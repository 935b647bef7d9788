"""Measurements of test_gpu_fit_scale.py, importable and runnable in a fresh process (the KBO_FIT_* schedule switches are read
once per process).  One fit of a history at production N, its factors checked on the GPU against an FP64 Gram matrix rebuilt
here by exact differences (as oracle.kernel_matrix forms it) and against a LAPACK reference saved by the caller; only numbers
come back: per-256×256-tile worst errors and where they are, the suggestion, a SHA-256 of L.  `current` runs the same checks
on whatever an engine holds after kbo_fit_append / kbo_fit_rebase chains (test_gpu_append_scale.py).

    python tests/_fit_scale.py '<json spec>' out.json
spec: {"fits": [[N, case, var_mode, ref_prefix], ...]}  or  {"digests": [[N, var_mode], ...]}
      or  {"pivots": [[N, p], ...], "var_mode": "f64"|"tc"}
"""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gp_oracle as O             # noqa: E402  (tests/ may use the oracle's workload generators)
from kubeflow_b200 import _lib as Lb          # noqa: E402
from kubeflow_b200.gp import GPEngine         # noqa: E402

TILE = 256          # = the factorisation's panel width: a tile (i, j) names panel row i, panel column j
M_CAND = 4096

# the histories at production N: cfg3's θ of record (Matérn-5/2, D = 32), an isotropic RBF at D = 100, an ARD Matérn at D = 17
CASES = {"m32": dict(D=32, kind="matern52", ard=False), "r100": dict(D=100, kind="rbf", ard=False),
         "m17ard": dict(D=17, kind="matern52", ard=True)}


def history(N, case, M=M_CAND):
    c = CASES[case]
    X, y, Xc = O.synthetic(N, M, c["D"])
    th = dict(kind=c["kind"], **O.theta_of_record(c["D"]))
    if c["ard"]:
        th["length_scale"] = th["length_scale"] * np.linspace(0.6, 1.5, c["D"])
    return X, y, Xc, th


def engine(th, var_mode, **kw):
    return GPEngine(0, kernel=th["kind"], acq="ei", var_mode=var_mode, length_scale=th["length_scale"], amplitude=th["amplitude"],
                    noise=th["noise"], xi=th["xi"], kappa=th["kappa"], **kw)


def gram(X, th):
    """amplitude·k(X, X) + noise·I in FP64 on the GPU, squared distances by exact differences (scipy cdist's arithmetic)."""
    Xs = torch.tensor(np.asarray(X) / th["length_scale"], device="cuda")
    N = Xs.shape[0]
    K = torch.empty(N, N, dtype=torch.float64, device="cuda")
    for r0 in range(0, N, 64):
        d2 = ((Xs[r0:r0 + 64, None, :] - Xs[None, :, :]) ** 2).sum(-1)
        if th["kind"] == "rbf":
            k = torch.exp(-0.5 * d2)
        else:
            s = torch.sqrt(5.0 * d2)
            k = (1.0 + s + s * s / 3.0) * torch.exp(-s)
        K[r0:r0 + 64] = th["amplitude"] * k
    K.diagonal().add_(th["noise"])
    return K


def fit_info(e):
    """(status, info) of kbo_fit_info: the Python wrapper raises on a failed fit before the pivot index can be read."""
    inf = C.c_int32()
    rc = e.lib.kbo_fit_info(e._h, None, None, None, None, C.byref(inf), e._stream())
    return rc, inf.value


def state(e, with_w=True):
    """L, W (None: not asked for — a lazy fit's missing rows are then not formed) and alpha, as kbo_fit_state returns them."""
    N = e.N
    Lm = torch.empty(N, N, dtype=torch.float64, device="cuda")
    Wm = torch.empty(N, N, dtype=torch.float64, device="cuda") if with_w else None
    al = torch.empty(N, dtype=torch.float64, device="cuda")
    rc = e.lib.kbo_fit_state(e._h, Lm.data_ptr(), Wm.data_ptr() if with_w else None, al.data_ptr(), e._stream())
    Lb.check(e.lib, e._h, rc)
    torch.cuda.synchronize()
    return Lm, Wm, al


def tile_max(E):
    """Largest |E| and the (row, column) of the 256×256 tile holding it."""
    n = E.shape[0]
    nb = (n + TILE - 1) // TILE
    pad = nb * TILE - n
    m = torch.nn.functional.pad(E.abs(), (0, pad, 0, pad)).view(nb, TILE, nb, TILE).amax(dim=(1, 3))
    v, i = m.flatten().max(0)
    return float(v), tuple(divmod(int(i), nb))


def device_y_stats(y):
    """y_mean / y_opt exactly as the fit's one-CTA reduction forms them (1024 strided partial sums, then a halving tree)."""
    a = np.zeros(1024)
    for k in range(0, len(y), 1024):
        part = y[k:k + 1024]
        a[:len(part)] += part
    o = 512
    while o:
        a[:o] += a[o:2 * o]
        o //= 2
    return a[0] / len(y), float(np.min(y))


def lapack(X, y, th):
    """oracle.gp_fit of a history (scipy cholesky / cho_solve) with cond_lb, the bound the forward errors are scaled by."""
    f = O.gp_fit(X, y, kind=th["kind"], length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    d = np.diag(f["L"])
    f["cond_lb"] = float((th["amplitude"] + th["noise"]) / d.min() ** 2)   # 1/λ_min >= 1/min pivot: a lower bound on cond(K)
    return f


def reference(N, case, prefix):
    """LAPACK factor of the history (oracle.gp_fit: scipy cholesky / cho_solve) -> prefix_L.npy, prefix_alpha.npy and the scalars."""
    X, y, _, th = history(N, case, M=1)
    f = lapack(X, y, th)
    np.save(prefix + "_L.npy", f["L"])
    np.save(prefix + "_alpha.npy", f["alpha"])
    return dict(lml=f["lml"], y_mean=f["y_mean"], y_std=f["y_std"], cond_lb=f["cond_lb"])


def _errors(K, Lm, Wm, al, yn, Lref, aref, tag="", first=None):
    """`first`: also the worst entry in rows [first, N) of K − LLᵀ and WL − I — the rows kbo_fit_append bordered on."""
    r = {}
    kmax = float(K.diagonal().max())
    E = K - Lm @ Lm.T
    r["backward" + tag], r["backward_tile" + tag] = tile_max(E)
    r["backward" + tag] /= kmax
    if first is not None:
        r["backward_app" + tag] = float(E[first:].abs().max()) / kmax
    del E
    r["upper_L_nonzero" + tag] = int(torch.count_nonzero(torch.triu(Lm, 1)))
    r["alpha_res" + tag] = float(torch.linalg.vector_norm(K @ al - yn) / (torch.linalg.matrix_norm(K) * torch.linalg.vector_norm(al)))
    r["L_fwd" + tag] = float((Lm - Lref).abs().max() / Lref.abs().max())
    r["alpha_fwd" + tag] = float((al - aref).abs().max() / aref.abs().max())
    if Wm is not None:
        I = torch.eye(K.shape[0], dtype=torch.float64, device="cuda")
        E = Wm @ Lm - I
        r["WL" + tag], r["WL_tile" + tag] = tile_max(E)
        if first is not None:
            r["WL_app" + tag] = float(E[first:].abs().max())
        del E
        r["LW" + tag], r["LW_tile" + tag] = tile_max(Lm @ Wm - I)
        r["upper_W_nonzero" + tag] = int(torch.count_nonzero(torch.triu(Wm, 1)))
    return r


def current(e, X, y, th, ref, first=None):
    """The checks of `measure` on whatever the engine holds now — after kbo_fit_append / kbo_fit_rebase chains too — against a
    Gram matrix rebuilt from (X, y) and its LAPACK factor `ref` (`lapack`).  `first`: the first appended row, whose rows are
    also reported on their own."""
    fi = e.fit_info()
    assert e.N == len(y), (e.N, len(y))
    K = gram(X, th)
    Lm, Wm, al = state(e)
    yn = torch.tensor((y - fi["y_mean"]) / fi["y_std"], device="cuda")
    Lref, aref = torch.tensor(ref["L"], device="cuda"), torch.tensor(ref["alpha"], device="cuda")
    r = dict(N=e.N, info=fi["info"], lml=fi["lml"], y_mean=fi["y_mean"], y_std=fi["y_std"], y_opt=fi["y_opt"],
             pivot_last=float(Lm[-1, -1]))
    r.update(_errors(K, Lm, Wm, al, yn, Lref, aref, first=first))
    del K, Lm, Wm, al, Lref, aref
    torch.cuda.empty_cache()
    return r


def measure(N, case, var_mode, prefix):
    """One fit: every error of §factors against the FP64 Gram matrix and the LAPACK reference at `prefix`, the LML, y statistics,
    the suggestion on M_CAND candidates and SHA-256 of L.  A tensor-core fit is checked before and after its lazy inverse is formed."""
    X, y, Xc, th = history(N, case)
    e = engine(th, var_mode)
    e.tell(X, y)
    rc, info = fit_info(e)
    fi = e.fit_info() if rc == 0 else dict(lml=float("nan"), y_mean=float("nan"), y_std=float("nan"), y_opt=float("nan"))
    b = e.ask(Xc)
    K = gram(X, th)
    Lref = torch.tensor(np.load(prefix + "_L.npy"), device="cuda")
    aref = torch.tensor(np.load(prefix + "_alpha.npy"), device="cuda")
    yn = torch.tensor((y - fi["y_mean"]) / fi["y_std"], device="cuda")
    r = dict(N=N, case=case, var_mode=var_mode, info=info, lml=fi["lml"], y_mean=fi["y_mean"], y_std=fi["y_std"], y_opt=fi["y_opt"],
             index=b.index, value=b.value, mu=b.mu, std=b.std, lazy=var_mode == "tc")
    if var_mode == "tc":
        Lm, _, al = state(e, with_w=False)    # L and the z-solve's alpha, the inverse's missing rows not formed yet
        r.update(_errors(K, Lm, None, al, yn, Lref, aref, "_lazy"))
        r["sha_L_lazy"] = hashlib.sha256(torch.tril(Lm).cpu().numpy().tobytes()).hexdigest()
        del Lm, al
    Lm, Wm, al = state(e)
    r.update(_errors(K, Lm, Wm, al, yn, Lref, aref))
    r["sha_L"] = hashlib.sha256(torch.tril(Lm).cpu().numpy().tobytes()).hexdigest()
    e.close()
    del K, Lm, Wm, al, Lref, aref
    torch.cuda.empty_cache()
    return r


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def digests(N, var_mode, case="m32"):
    """SHA-256 of everything one fit and one suggestion produce, bit for bit: tril(L) and alpha (a tensor-core fit's before the
    rest of W is formed), the LML and y statistics, the suggestion over M_CAND candidates, and W for an FP64 fit."""
    X, y, Xc, th = history(N, case)
    e = engine(th, var_mode)
    e.tell(X, y)
    Lm, _, al = state(e, with_w=False)
    r = dict(L=_sha(torch.tril(Lm).cpu().numpy()), alpha=_sha(al.cpu().numpy()))
    del Lm, al
    fi = e.fit_info()
    r["fit"] = _sha(np.array([fi["lml"], fi["y_mean"], fi["y_std"], fi["y_opt"]], dtype=np.float64))
    b = e.ask(Xc)
    r["ask"] = _sha(np.array([b.index], dtype=np.int64), np.array([b.value, b.mu, b.std], dtype=np.float64))
    if var_mode == "f64":
        r["W"] = _sha(torch.tril(state(e)[1]).cpu().numpy())
    e.close()
    torch.cuda.empty_cache()
    return r


def pivot_engine(var_mode):
    """RBF, amplitude 1, ℓ = 1, noise 0: the θ under which oracle.not_pd_at's histories fail at exactly the chosen pivot."""
    return GPEngine(0, kernel="rbf", acq="ei", var_mode=var_mode, length_scale=1.0, amplitude=1.0, noise=0.0)


def pivot_report(e, X):
    """What a failed fit reports: info, and the status of every call that needs a factorisation."""
    Xc = np.random.default_rng(5).random((512, X.shape[1])) * 16.0
    rc, info = fit_info(e)
    out = dict(fit_info_rc=rc, info=info)
    for name, call in (("ask", lambda: e.ask(Xc)), ("ask_multi", lambda: e.ask_multi(Xc, ["ei", "lcb"])),
                       ("predict_mean", lambda: e.predict_mean(Xc[:7])), ("lml_grad", lambda: e.lml_grad())):
        try:
            call()
            out[name] = "ok"
        except Lb.KboNotPositiveDefinite:
            out[name] = "not_pd"
        except Lb.KboError as ex:
            out[name] = f"error {ex.code}"
    g = np.empty(3, dtype=np.float64)
    out["abi_lml_grad_rc"] = int(e.lib.kbo_lml_grad(e._h, g.ctypes.data_as(C.POINTER(C.c_double)), 3, e._stream()))
    return out


def pivots(cases, var_mode):
    res = []
    for N, p in cases:
        X, y = O.not_pd_at(N, p)
        e = pivot_engine(var_mode)
        e.tell(X, y)
        res.append(dict(N=N, p=p, var_mode=var_mode, **pivot_report(e, X)))
        e.close()
    return res


if __name__ == "__main__":
    spec, out = json.loads(sys.argv[1]), sys.argv[2]
    if "fits" in spec:
        res = [measure(N, case, vm, prefix) for N, case, vm, prefix in spec["fits"]]
    elif "digests" in spec:
        res = [digests(N, vm) for N, vm in spec["digests"]]
    else:
        res = pivots(spec["pivots"], spec["var_mode"])
    with open(out, "w") as f:
        json.dump(res, f)
