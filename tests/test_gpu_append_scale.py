"""kbo_fit_append and kbo_fit_rebase at the history sizes and stack depths the service reaches, in f64, tc and auto mode.

A running Katib experiment rarely refits: each GetSuggestions request drops the last constant-liar rows (kbo_fit_rebase) and
appends the finished trials and the new lies (kbo_fit_append).  After a chain, the engine's factors are checked as
test_gpu_fit_scale.py checks a fit — against an FP64 Gram matrix rebuilt from the extended history and its LAPACK factor —
and its suggestions against a fresh kbo_fit of the same rows.

Tolerances are 4× the worst value measured on one H100 80GB HBM3 (400 W power limit) over every case below (worst seen in
brackets); the suggestion's value keeps the 1e-10 of the other suggestion tests, the auto-mode arrays the bounds of
test_gpu_theta_range.py (1e-6 on μ, 1e-5 on EI).
  |K − LLᵀ|/max K per tile, and in the appended rows   5.1e-14  (1.26e-14: ARD Matérn D = 17, 5800 + 24; rows 9.4e-15)
  |WL − I|, |LW − I| per tile, and in the appended rows 6.1e-14  (1.52e-14: Matérn D = 32, 8129 + 63; rows 8.8e-15)
  |Kα − yn| / (|K|_F |α|)                               1.9e-16  (4.7e-17)
  |L − L_LAPACK| / max|L_LAPACK|                        28 eps·cond_lb   (6.8)
  |α − α_cho_solve| / max|α_cho_solve|                  465 eps·cond_lb  (116)
  LML against gp_fit                                    4.3e-14 relative (1.07e-14)
  kbo_lml_grad against the oracle                       6.7e-14 of max|g| (1.7e-14)
  μ, σ of the suggestion against a fresh fit            7.4e-13 (1.8e-13)
  near duplicates: appended pivot against LAPACK's      23 eps·(amp + noise)/d² relative (5.8); its row 4.1 eps·cond_lb (1.0)

Stack depth: S rows appended on a fit of 4096 + S rows rebased to 4096 (Matérn D = 32), the worst entry in the appended rows
against a fresh fit's worst tile on the same history, f64 and tc alike:
              S = 63               S = 255              S = 511              fresh fit
  noise 1e-3  6.7e-15  WL 5.5e-15  7.4e-15  WL 5.5e-15  8.4e-15  WL 6.3e-15  9.1e-15  WL 7.6e-15   (|K − LLᵀ|/max K, |WL − I|)
  noise 1e-6  7.4e-15  WL 4.7e-15  7.4e-15  WL 6.5e-15  7.5e-15  WL 6.7e-15  8.0e-15  WL 1.1e-14
The error does not grow with the depth and stays below the fresh fit's, and every suggestion is the fresh fit's, so the
stack is bounded by the fit's row pitch alone (kbo_fit_room = pitch − N).
"""
import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky

from oracle import gp_oracle as O
from tests import _fit_scale as H

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
TOL_BWD = 5.1e-14     # |K − LLᵀ|/max K, per tile and in the appended rows
TOL_WINV = 6.1e-14    # |WL − I|, |LW − I|
TOL_ARES = 1.9e-16    # |Kα − yn| / (|K|_F |α|)
TOL_LFWD = 28.0       # |L − L_LAPACK| / max|L_LAPACK|, in eps·cond_lb
TOL_AFWD = 465.0      # |α − α_cho_solve| / max|α_cho_solve|, in eps·cond_lb
TOL_LML = 4.3e-14     # LML against LAPACK's, relative
TOL_GRAD = 6.7e-14    # kbo_lml_grad against the row-chunked oracle, of max|g|
TOL_PIVOT = 23.0      # |d − d_LAPACK| / d_LAPACK of an appended pivot, in eps·(amplitude + noise)/d²
TOL_ROW = 4.1         # |l − l_LAPACK| / max|l_LAPACK| of an appended row, in eps·cond_lb
TOL_VALUE = 1e-10     # suggestion value against a fresh fit's, relative
TOL_MS = 7.4e-13      # μ and σ of the suggestion against a fresh fit's, relative to max(1, |·|)
M_AUTO = 262144       # M·N² > 2e11 at N = 1000: auto mode's tensor-core threshold


@pytest.fixture(scope="module")
def lapack():
    """LAPACK factors, one per history, shared by every var_mode that runs a chain on it."""
    cache = {}

    def get(key, X, y, th):
        if key not in cache:
            cache[key] = H.lapack(X, y, th)
        return cache[key]
    return get


def _print(name, r):
    keys = [k for k in ("backward", "backward_app", "WL", "WL_app", "LW", "alpha_res") if k in r]
    print(f"\n[{name}] " + " ".join(f"{k}={r[k]:.3e}" for k in keys)
          + f" L_fwd/eps.cond={r['L_fwd_u']:.3f} alpha_fwd/eps.cond={r['alpha_fwd_u']:.3f} dlml={r['dlml']:.2e}")


def _check_factors(name, r, ref, X, y):
    """Every check of test_gpu_fit_scale._check on a chain's state, the appended rows on their own, and the y statistics."""
    r["L_fwd_u"], r["alpha_fwd_u"] = r["L_fwd"] / (EPS * ref["cond_lb"]), r["alpha_fwd"] / (EPS * ref["cond_lb"])
    r["dlml"] = abs(r["lml"] - ref["lml"]) / abs(ref["lml"])
    _print(name, r)
    assert r["info"] == 0, name
    assert r["backward"] <= TOL_BWD, f"{name}: |K − LLᵀ| {r['backward']:.3e} in tile {r['backward_tile']}"
    assert r.get("backward_app", 0.0) <= TOL_BWD, f"{name}: |K − LLᵀ| {r['backward_app']:.3e} in the appended rows"
    for key in ("WL", "LW"):
        assert r[key] <= TOL_WINV, f"{name}: |{key} − I| {r[key]:.3e} in tile {r[key + '_tile']}"
    assert r.get("WL_app", 0.0) <= TOL_WINV, f"{name}: |WL − I| {r['WL_app']:.3e} in the appended rows"
    assert r["upper_L_nonzero"] == 0 and r["upper_W_nonzero"] == 0, (name, r["upper_L_nonzero"], r["upper_W_nonzero"])
    assert r["alpha_res"] <= TOL_ARES, f"{name}: |Kα − yn|/(|K||α|) {r['alpha_res']:.3e}"
    assert r["L_fwd_u"] <= TOL_LFWD, f"{name}: L vs LAPACK {r['L_fwd_u']:.2f}·eps·cond_lb (cond_lb {ref['cond_lb']:.3e})"
    assert r["alpha_fwd_u"] <= TOL_AFWD, f"{name}: alpha vs cho_solve {r['alpha_fwd_u']:.2f}·eps·cond_lb"
    assert r["dlml"] <= TOL_LML, f"{name}: LML {r['lml']!r} vs gp_fit {ref['lml']!r}"
    ym, yo = H.device_y_stats(y)
    assert r["y_mean"] == ym and r["y_opt"] == yo, (name, r["y_mean"], ym, r["y_opt"], yo)
    assert abs(r["y_std"] - ref["y_std"]) <= 4 * EPS * ref["y_std"], (name, r["y_std"], ref["y_std"])


def _same_best(name, b, bf):
    msg = f"{name}: index {b.index} value {b.value!r} mu {b.mu!r} std {b.std!r}; fresh {bf.index} {bf.value!r} {bf.mu!r} {bf.std!r}"
    assert b.index == bf.index and abs(b.value - bf.value) <= TOL_VALUE * max(1.0, abs(bf.value)), msg
    assert abs(b.mu - bf.mu) <= TOL_MS * max(1.0, abs(bf.mu)) and abs(b.std - bf.std) <= TOL_MS * max(1.0, abs(bf.std)), msg


def _against_fresh(name, e, X, y, th, var_mode, Xc, multi=True):
    """The chain's suggestion (and gp_hedge's three) against a fresh kbo_fit of the same history in the same mode."""
    f = H.engine(th, var_mode)
    f.tell(X, y)
    b, bf = e.ask(Xc), f.ask(Xc)
    print(f"    [{name}] suggestion {b.index} {b.value!r}; fresh {bf.index} {bf.value!r} (d = {b.value - bf.value:.2e}, "
          f"d mu {b.mu - bf.mu:.2e}, d std {b.std - bf.std:.2e})")
    _same_best(name, b, bf)
    if multi:
        for a, (m, mf) in zip(("ei", "lcb", "pi"), zip(e.ask_multi(Xc, ["ei", "lcb", "pi"]), f.ask_multi(Xc, ["ei", "lcb", "pi"]))):
            _same_best(f"{name} ask_multi {a}", m, mf)
    f.close()


def _lies(n, D, y, seed):
    """Stand-in constant-liar rows: n points the real history does not have, at cl_min's target."""
    return np.random.default_rng(seed).random((n, D)), np.full(n, float(np.min(y)))


def _append(e, X, y, lo, hi):
    assert e.room() >= hi - lo, (e.room(), hi - lo)
    for i in range(lo, hi):
        e.append(X[i], y[i])


# ---- 1. append chains at production N -------------------------------------------------------------------------------------
def _chain(name, var_mode):
    """-> (engine, X, y, Xc, th, first appended row) after the chain."""
    if name == "fill-pitch-8192":        # cfg3's θ of record: fit 8129, append 63 — the whole 64-row pitch
        X, y, Xc, th = H.history(8192, "m32")
        e = H.engine(th, var_mode)
        e.tell(X[:8129], y[:8129])
        _append(e, X, y, 8129, 8192)
        return e, X, y, Xc, th, 8129
    if name == "rebase-4200-4090-4224":  # Npad 4096 -> 4352; the pruning prefix P1 goes from 1 to 2 tile pairs
        X, y, Xc, th = H.history(4224, "m32")
        Xl, yl = _lies(110, 32, y[:4090], 21)
        e = H.engine(th, var_mode)
        e.tell(np.vstack([X[:4090], Xl]), np.concatenate([y[:4090], yl]))
        e.rebase(4090)
        _append(e, X, y, 4090, 4224)
        return e, X, y, Xc, th, 4090
    assert name == "ard17-5800-5824"     # a lazy tensor-core fit: the first append forms the rest of W
    X, y, Xc, th = H.history(5824, "m17ard")
    e = H.engine(th, var_mode)
    e.tell(X[:5800], y[:5800])
    _append(e, X, y, 5800, 5824)
    return e, X, y, Xc, th, 5800


@pytest.mark.parametrize("var_mode", ["f64", "tc", "auto"])
@pytest.mark.parametrize("name", ["fill-pitch-8192", "rebase-4200-4090-4224", "ard17-5800-5824"])
def test_append_chain_at_production_n_against_lapack(name, var_mode, lapack):
    """After each chain: backward errors per tile and in the appended rows, strict upper triangles zero, the residual of α, L
    and α against LAPACK, the LML, y statistics bit for bit; the suggestion and gp_hedge's three against a fresh fit."""
    e, X, y, Xc, th, first = _chain(name, var_mode)
    ref = lapack(name, X, y, th)
    r = H.current(e, X, y, th, ref, first)
    _check_factors(f"{name} {var_mode}", r, ref, X, y)
    if name.startswith("ard17"):
        _, g = e.lml_grad()
        _, ref_g = O.lml_and_grad(X, y, kind=th["kind"], length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
        err = np.abs(g - ref_g).max() / np.abs(ref_g).max()
        print(f"    lml_grad |g − oracle|/max|g| {err:.3e}")
        assert err <= TOL_GRAD, err
    _against_fresh(f"{name} {var_mode}", e, X, y, th, var_mode, Xc)
    e.close()


# ---- 2. stack depth: fit N0 + S (S lies), rebase to N0, append S real rows -----------------------------------------------------
N0 = 4096


@pytest.mark.parametrize("var_mode", ["f64", "tc"])
@pytest.mark.parametrize("noise", [1e-3, 1e-6])
@pytest.mark.parametrize("S", [63, 255, 511])
def test_stack_depth_after_a_rebase(S, noise, var_mode, lapack):
    """A rebase keeps the pitch of the fit it shrinks, so kbo_fit_room() is ld − N0 and up to S rows stack on a factor that is
    never refreshed, each formed from the W rows of the appends before it.  The appended rows against the fit's bounds and
    against a fresh fit of the same history."""
    X, y, Xc, th = H.history(N0 + S, "m32")
    th = dict(th, noise=noise)
    Xl, yl = _lies(S, 32, y[:N0], 31)
    e = H.engine(th, var_mode)
    e.tell(np.vstack([X[:N0], Xl]), np.concatenate([y[:N0], yl]))
    e.rebase(N0)
    _append(e, X, y, N0, N0 + S)
    ref = lapack(("stack", S, noise), X, y, th)
    name = f"stack S={S} noise={noise:g} {var_mode}"
    r = H.current(e, X, y, th, ref, N0)
    f = H.engine(th, "f64")
    f.tell(X, y)
    rf = H.current(f, X, y, th, ref)
    print(f"\n[{name}] appended rows: |K − LLᵀ| {r['backward_app']:.3e} |WL − I| {r['WL_app']:.3e}; fresh fit worst tile: "
          f"{rf['backward']:.3e} {rf['WL']:.3e}; ratio {r['backward_app'] / rf['backward']:.2f} {r['WL_app'] / rf['WL']:.2f}")
    f.close()
    _check_factors(name, r, ref, X, y)
    _against_fresh(name, e, X, y, th, var_mode, Xc, multi=False)
    e.close()


# ---- 3. near duplicates ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise", [1e-6, 1e-3])
def test_near_duplicate_append(noise):
    """x_j + δ·ℓ·u appended to a fitted history at N = 4096: the Schur complement is at least the noise, so never NOT_PD; the
    pivot and the row against LAPACK's factor of the extended matrix; the tensor-core suggestion (whose fp16 scale the new
    W row drives) against the FP64 engine's."""
    X, y, _, th = H.history(N0, "m32")
    th = dict(th, noise=noise)
    Xl, yl = _lies(1, 32, y, 37)         # a fit of N0 rows fills its pitch: fit one more and rebase, for room to append
    Xc = O.synthetic(1, 30000, 32)[2]
    j = 1234
    u = np.random.default_rng(41).standard_normal(32)
    u /= np.linalg.norm(u)
    Xc[:16] = X[j] + 0.2 * th["length_scale"] * np.random.default_rng(43).standard_normal((16, 32)) / np.sqrt(32)   # near x_j too
    K = O.kernel_matrix(X, X, th["length_scale"], th["kind"], th["amplitude"])
    K[np.diag_indices_from(K)] += noise
    engs = {m: H.engine(th, m) for m in ("f64", "tc")}
    for e in engs.values():
        e.tell(np.vstack([X, Xl]), np.concatenate([y, yl]))
        e.rebase(N0)
    for delta in (1e-1, 1e-3, 1e-5):
        x = X[j] + delta * th["length_scale"] * u
        k = O.kernel_matrix(x[None], X, th["length_scale"], th["kind"], th["amplitude"])[0]
        Kx = np.block([[K, k[:, None]], [k[None, :], np.array([[th["amplitude"] + noise]])]])
        Lx = cholesky(Kx, lower=True, check_finite=False)
        d_ref, l_ref = Lx[-1, -1], Lx[-1, :-1]
        cond_lb = (th["amplitude"] + noise) / np.diag(Lx).min() ** 2
        bests = {}
        for m, e in engs.items():
            e.append(x, y[j])
            assert H.fit_info(e) == (0, 0), (m, delta, noise)
            Lm, _, _ = H.state(e, with_w=False)
            row = Lm[-1].cpu().numpy()
            d = row[N0]
            bwd = float(np.abs(Kx[-1] - Lm.cpu().numpy() @ row).max()) / (th["amplitude"] + noise)
            dp = abs(d - d_ref) / d_ref / (EPS * (th["amplitude"] + noise) / d_ref ** 2)
            dl = np.abs(row[:N0] - l_ref).max() / np.abs(l_ref).max() / (EPS * cond_lb)
            bests[m] = e.ask(Xc)
            print(f"\n[near duplicate δ={delta:g} noise={noise:g} {m}] d {d:.6e} (LAPACK {d_ref:.6e}) |Δd|/d {dp:.3f}·eps·(amp+noise)/d² "
                  f"row {dl:.3f}·eps·cond_lb |K − LLᵀ| last row {bwd:.3e}; suggestion {bests[m].index} {bests[m].value!r} "
                  f"unrefined {e.last_unrefined()}")
            assert dp <= TOL_PIVOT and dl <= TOL_ROW and bwd <= TOL_BWD, (m, delta, noise, dp, dl, bwd)
            del Lm
        b, b6 = bests["tc"], bests["f64"]
        assert b.index == b6.index and abs(b.value - b6.value) <= TOL_VALUE * max(1.0, abs(b6.value)), (delta, noise, b, b6)
        assert engs["tc"].last_unrefined() == 0
        for e in engs.values():
            e.rebase(N0)
    for e in engs.values():
        e.close()


# ---- 4. auto mode across N = 1024 -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_app", [0, 10, 30])
def test_auto_mode_after_a_rebase_below_1024(n_app):
    """Fit 1100 rows (100 lies) in auto mode — N > 1024 builds the fp16 planes of W — rebase to 1000, append n_app rows, sweep
    M = 262144 candidates (M·N² > 2e11: auto's tensor-core threshold).  At N ≤ 1024 auto builds no planes, so the sweep must not
    contract with the 1100-row fit's (their row stride is the old Npad); at 1030 they are rebuilt.  Array-free suggestion and
    arrays against a fresh auto fit and the FP64 engine."""
    D = 6
    X, y, Xc = O.synthetic(1000 + n_app, M_AUTO, D)
    th = dict(kind="matern52", **O.theta_of_record(D))
    Xl, yl = _lies(100, D, y[:1000], 51)
    e = H.engine(th, "auto")
    e.tell(np.vstack([X[:1000], Xl]), np.concatenate([y[:1000], yl]))
    e.rebase(1000)
    _append(e, X, y, 1000, 1000 + n_app)
    fresh, f64 = H.engine(th, "auto"), H.engine(th, "f64")
    fresh.tell(X, y)
    f64.tell(X, y)
    b, bf, b6 = e.ask(Xc), fresh.ask(Xc), f64.ask(Xc)
    _, mu, sd, a = e.ask(Xc, return_arrays=True)
    arrays = {k: g.ask(Xc, return_arrays=True)[1:] for k, g in (("fresh auto", fresh), ("f64", f64))}
    name = f"auto 1100 -> 1000 -> {1000 + n_app}"
    for k, (mu_r, sd_r, a_r) in arrays.items():
        dm, ds, da = (float((p - q).abs().max()) for p, q in ((mu, mu_r), (sd, sd_r), (a, a_r)))
        print(f"\n[{name}] against {k}: max|d mu| {dm:.3e} max|d std| {ds:.3e} max|d ei| {da:.3e}")
        assert dm <= 1e-6 and da <= 1e-5, (name, k, dm, ds, da)
    print(f"    suggestion {b.index} {b.value!r}; fresh auto {bf.index} {bf.value!r}; f64 {b6.index} {b6.value!r}")
    _same_best(f"{name} vs fresh auto", b, bf)
    _same_best(f"{name} vs f64", b, b6)
    for g in (e, fresh, f64):
        g.close()


def test_optimizer_incremental_across_1024_suggests_what_a_refit_does():
    """The service's default Optimizer (incremental, auto) with n_points = 262144 and a history of 1000: the lies of the first
    request refit past 1024 (planes built), the second request reports 10 of the 40 and rebases to 1010.  Its 80 points must be
    the refitting Optimizer's; where they differ, the two must tie in EI within 1e-9 on the history they were asked on."""
    from kubeflow_b200.optimizer import Optimizer
    from kubeflow_b200.space import Real
    D = 6
    dims = [Real(0.0, 1.0, name=f"x{i}") for i in range(D)]

    def f(P):
        P = np.asarray(P, dtype=np.float64)
        return np.sin(3.0 * P.sum(axis=1) / np.sqrt(D)) + 0.5 * (P[:, 0] - 0.3) ** 2

    X0 = np.random.default_rng(61).random((1000, D))
    y0 = f(X0)
    runs, logs = {}, {}
    for inc in (True, False):
        opt = Optimizer(dims, n_initial_points=5, random_state=13, n_points=M_AUTO, incremental=inc)
        log = logs[inc] = []
        tell_engine = opt._tell_engine

        def rec(eng, Xt, ya, _t=tell_engine, _o=opt, _l=log):
            _t(eng, Xt, ya)
            _l.append((_o.last_fit, eng.N))
        opt._tell_engine = rec
        opt.tell(X0.tolist(), y0.tolist())
        a = opt.ask(n_points=40)
        opt.tell(a[:10], f(a[:10]).tolist())
        b = opt.ask(n_points=40)
        runs[inc] = [np.asarray(a), np.asarray(b)]
        opt._engine.close()
    assert ("rebase", 1010) in logs[True], logs[True][:45]
    told = [(X0, y0), (np.vstack([X0, runs[True][0][:10]]), np.concatenate([y0, f(runs[True][0][:10])]))]
    th = O.theta_of_record(D)
    for r in range(2):
        P, Q = runs[True][r], runs[False][r]
        diff = np.flatnonzero((P != Q).any(axis=1))
        print(f"\n[optimizer request {r + 1}] {len(diff)} of 40 points differ" + (f", first at {diff[0]}" if len(diff) else ""))
        if len(diff):
            i = int(diff[0])
            Xh = np.vstack([told[r][0], P[:i]])
            yh = np.concatenate([told[r][1], np.full(i, told[r][1].min())])
            fit = O.gp_fit(Xh, yh, kind="matern52", length_scale=th["length_scale"], amplitude=1.0, noise=1e-3)
            mu, sd = O.gp_predict(fit, np.vstack([P[i], Q[i]]))
            ei = O.acquisition(mu, sd, float(yh.min()), "ei", 0.01, 1.96)
            print(f"    EI at the two points {ei[0]!r} {ei[1]!r}")
            assert abs(ei[0] - ei[1]) <= 1e-9 * max(1.0, abs(ei[1])), (r, i, ei)
            break


# ---- 5. y-only rebase at 8192 ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("var_mode", ["f64", "tc"])
def test_y_only_rebase_at_8192(var_mode, lapack):
    """rebase(8192, y2): every trial's target replaced, L and W kept.  α and the LML against LAPACK's factor solved with y2, the
    suggestion against a fresh fit of (X, y2)."""
    X, y, Xc, th = H.history(8192, "m32")
    y2 = 2.5 * np.cos(5.0 * X[:, 0]) - y + 0.3
    ref = lapack("fill-pitch-8192", X, y, th)
    e = H.engine(th, var_mode)
    e.tell(X, y)
    e.rebase(8192, y2)
    fi = e.fit_info()
    yn = (y2 - y2.mean()) / y2.std()
    aref = cho_solve((ref["L"], True), yn, check_finite=False)
    lml_ref = float(-0.5 * yn @ aref - np.log(np.diag(ref["L"])).sum() - 0.5 * len(yn) * np.log(2 * np.pi))
    _, _, al = H.state(e, with_w=False)
    al = al.cpu().numpy()
    af = np.abs(al - aref).max() / np.abs(aref).max() / (EPS * ref["cond_lb"])
    dl = abs(fi["lml"] - lml_ref) / abs(lml_ref)
    ym, yo = H.device_y_stats(y2)
    print(f"\n[y-only rebase 8192 {var_mode}] alpha_fwd/eps.cond={af:.3f} dlml={dl:.2e}")
    assert fi["info"] == 0 and fi["y_mean"] == ym and fi["y_opt"] == yo
    assert af <= TOL_AFWD and dl <= TOL_LML, (af, dl)
    _against_fresh(f"y-only rebase 8192 {var_mode}", e, X, y2, th, var_mode, Xc, multi=False)
    e.close()
