"""The fit at the history sizes it serves (N = 4096 … 8192: 16 to 32 panels, the SM partition on, the early-Gram path) against an
independent FP64 Gram matrix and LAPACK, in every factorisation schedule; kbo_lml_grad and kbo_lml_batch at the θ-search sizes;
and the non-positive-pivot report, on histories built to fail at an exact pivot.

Backward errors (|K − L·Lᵀ|, |W·L − I|, |L·W − I| per 256×256 tile, the residual of alpha) do not depend on conditioning: a
correct blocked FP64 Cholesky leaves ~1e-15 … 1e-14, a skipped or doubled tile update O(1) in the tiles it touched, and the
message names the worst tile as (panel row, panel column).  Forward errors against LAPACK scale with cond(K); they are held
relative to eps·cond_lb, cond_lb = (amplitude + noise)/min pivot² ≤ cond(K).

Tolerances are 4× the worst value measured on one H100 80GB HBM3 over every case and schedule below (worst seen in brackets):
  |K − LLᵀ|/max K per tile            5e-14   (1.26e-14: ARD Matérn D = 17, N = 5800; 1.20e-14 Matérn D = 32, N = 8192)
  |WL − I|, |LW − I| per tile          7e-14   (1.70e-14: RBF D = 100, N = 8192)
  |Kα − yn| / (|K|_F |α|)               1.5e-16 (3.7e-17)
  |L − L_LAPACK| / max|L_LAPACK|        32 eps·cond_lb  (7.9)
  |α − α_cho_solve| / max|α_cho_solve|  450 eps·cond_lb (111)
  LML against gp_fit                    1e-9 relative (1.3e-14 measured; 1.1e-12 for kbo_lml_batch at noise 3e-4)
  kbo_lml_grad against the oracle       1e-11 of max|g| (2.2e-12: RBF ARD D = 17, N = 4097)
  kbo_lml_grad against central differences of the engine's LML, step 2e-4 in log θ:
                                        1.8e-6 of max|g| (4.4e-7: RBF D = 33, N = 2048; truncation, O(step²))
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O
from tests import _fit_scale as H

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
TOL_BWD = 5e-14
TOL_WINV = 7e-14
TOL_ARES = 1.5e-16
TOL_LFWD = 32.0
TOL_AFWD = 450.0
TOL_LML = 1e-9
HELPER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_fit_scale.py")


@pytest.fixture(scope="module")
def refs(tmp_path_factory):
    """LAPACK references, computed once per history and shared by the in-process fits and the schedule subprocesses."""
    d = tmp_path_factory.mktemp("lapack")
    cache = {}

    def get(N, case):
        if (N, case) not in cache:
            prefix = str(d / f"{case}_{N}")
            cache[(N, case)] = (prefix, H.reference(N, case, prefix))
        return cache[(N, case)]
    return get


def _check(r, ref, where):
    """The checks of test_factors_at_production_sizes_against_lapack on one measurement `r` (H.measure) against its LAPACK reference."""
    name = f"{where} N={r['N']} {r['case']} {r['var_mode']}"
    assert r["info"] == 0, name
    for tag in (("_lazy", "") if r["lazy"] else ("",)):
        t = name + (" before the lazy inverse is formed" if tag else "")
        assert r["backward" + tag] <= TOL_BWD, f"{t}: |K − LLᵀ| {r['backward' + tag]:.3e} in tile {r['backward_tile' + tag]} > {TOL_BWD:.1e}"
        assert r["upper_L_nonzero" + tag] == 0, f"{t}: {r['upper_L_nonzero' + tag]} nonzeros above L's diagonal"
        assert r["alpha_res" + tag] <= TOL_ARES, f"{t}: |Kα − yn|/(|K||α|) {r['alpha_res' + tag]:.3e} > {TOL_ARES:.1e}"
        lf, af = r["L_fwd" + tag] / (EPS * ref["cond_lb"]), r["alpha_fwd" + tag] / (EPS * ref["cond_lb"])
        assert lf <= TOL_LFWD, f"{t}: L vs LAPACK {r['L_fwd' + tag]:.3e} = {lf:.2f}·eps·cond_lb (cond_lb {ref['cond_lb']:.3e}) > {TOL_LFWD}"
        assert af <= TOL_AFWD, f"{t}: alpha vs cho_solve {r['alpha_fwd' + tag]:.3e} = {af:.2f}·eps·cond_lb > {TOL_AFWD}"
    if r["lazy"]:
        assert r["sha_L"] == r["sha_L_lazy"], f"{name}: forming the rest of W changed L"
    for key in ("WL", "LW"):
        assert r[key] <= TOL_WINV, f"{name}: |{key} − I| {r[key]:.3e} in tile {r[key + '_tile']} > {TOL_WINV:.1e}"
    assert r["upper_W_nonzero"] == 0, f"{name}: {r['upper_W_nonzero']} nonzeros above W's diagonal"
    assert abs(r["lml"] - ref["lml"]) <= TOL_LML * abs(ref["lml"]), f"{name}: LML {r['lml']!r} vs gp_fit {ref['lml']!r}"


def _print(r, ref, where=""):
    keys = [k for k in ("backward_lazy", "backward", "WL", "LW", "alpha_res_lazy", "alpha_res") if k in r]
    print(f"\n[{where} N={r['N']} {r['case']} {r['var_mode']}] " + " ".join(f"{k}={r[k]:.3e}" for k in keys)
          + f" L_fwd/eps.cond={r['L_fwd'] / (EPS * ref['cond_lb']):.3f} alpha_fwd/eps.cond={r['alpha_fwd'] / (EPS * ref['cond_lb']):.3f}"
          + f" cond_lb={ref['cond_lb']:.3e} dlml={abs(r['lml'] - ref['lml']) / abs(ref['lml']):.2e}")


FACTOR_CASES = [(4096, "m32"), (5800, "m32"), (8191, "m32"), (8192, "m32"), (8192, "r100"), (5800, "m17ard")]


@pytest.mark.parametrize("var_mode", ["f64", "tc"])
@pytest.mark.parametrize("N,case", FACTOR_CASES)
def test_factors_at_production_sizes_against_lapack(N, case, var_mode, refs):
    """L, W = L⁻¹ and alpha of the default schedule: backward errors per tile, strict upper triangles exactly zero, L and alpha
    against scipy's cholesky / cho_solve, the LML against gp_fit, the y statistics as the device reduction forms them.  The
    tensor-core fit is lazy (only the leading rows of W): its L and its z-solve alpha are checked before and after the rest of W
    is formed."""
    prefix, ref = refs(N, case)
    r = H.measure(N, case, var_mode, prefix)
    _print(r, ref)
    _check(r, ref, "v3")
    X, y, _, _ = H.history(N, case, M=1)
    ym, yo = H.device_y_stats(y)
    assert r["y_mean"] == ym and r["y_opt"] == yo, (r["y_mean"], ym, r["y_opt"], yo)
    assert abs(r["y_mean"] - ref["y_mean"]) <= 4 * EPS * np.abs(y).max()
    assert abs(r["y_std"] - ref["y_std"]) <= 4 * EPS * ref["y_std"], (r["y_std"], ref["y_std"])


SCHEDULES = [("v3", {}), ("v3-unpartitioned", {"KBO_FIT_NO_PARTITION": "1"}), ("serial", {"KBO_FIT_SERIAL": "1"})]


def _helper(spec, out, env=None, timeout=600):
    subprocess.run([sys.executable, HELPER, json.dumps(spec), str(out)], check=True, env={**os.environ, **(env or {})}, timeout=timeout)
    with open(out) as f:
        return json.load(f)


def test_every_schedule_at_5800_and_8192_against_lapack(refs, tmp_path):
    """Each factorisation schedule in a fresh process (its switches are read once per process) at N = 5800 (23 panels: an odd
    count ends the merged bulk pairs early, a 40-row last block) as a lazy tensor-core fit and N = 8192 (32 panels) as an FP64
    fit: every check of the default schedule's test against the same LAPACK reference, and one suggestion for all."""
    fits = [(5800, "m32", "tc"), (8192, "m32", "f64")]
    spec = {"fits": [[N, case, vm, refs(N, case)[0]] for N, case, vm in fits]}
    runs = {}
    for name, env in SCHEDULES:
        runs[name] = _helper(spec, tmp_path / f"{name}.json", env)
        for r in runs[name]:
            _print(r, refs(r["N"], r["case"])[1], name)
    for name, rs in runs.items():
        for r, r0 in zip(rs, runs["v3"]):
            _check(r, refs(r["N"], r["case"])[1], name)
            assert r["index"] == r0["index"] and abs(r["value"] - r0["value"]) <= 1e-10 * max(1.0, abs(r0["value"])), \
                (name, r["N"], r["index"], r0["index"], r["value"], r0["value"])


# ---- LML gradient and batched LML at the θ-search sizes ------------------------------------------------------------------------
TOL_GRAD = 1e-11
TOL_FD = 1.8e-6


def _lml_history(N, D, kind, ard):
    X, y, _ = O.synthetic(N, 1, D)
    ls = 0.3 * np.sqrt(D) * (np.linspace(0.7, 1.4, D) if ard else 1.0)
    return X, y, dict(kind=kind, length_scale=ls, amplitude=1.3, noise=2e-3, xi=0.01, kappa=1.96)


@pytest.mark.parametrize("N,D,kind,ard,var_mode", [(2048, 17, "matern52", True, "f64"), (2048, 33, "rbf", False, "f64"),
                                                   (4097, 33, "matern52", True, "f64"), (4097, 17, "rbf", True, "f64"),
                                                   (4097, 17, "matern52", False, "f64"), (4097, 33, "rbf", True, "tc")])
def test_lml_grad_against_the_chunked_oracle_and_central_differences(N, D, kind, ard, var_mode):
    """kbo_lml_grad where its per-dimension sums run over several 16-wide D chunks (D = 17, 33), 33 to 65 pair-tile rows, a
    ragged last tile (4097) and a lazy tensor-core fit: against the row-chunked oracle, and against central differences of the
    engine's own FP64 LML in each log-θ component."""
    X, y, th = _lml_history(N, D, kind, ard)
    ref_lml, ref_g = O.lml_and_grad(X, y, kind=kind, length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    e = H.engine(th, var_mode)
    e.tell(X, y)
    lml, g = e.lml_grad()
    e.close()
    scale = np.abs(ref_g).max()
    err = np.abs(g - ref_g).max() / scale
    print(f"\n[lml_grad N={N} D={D} {kind} ard={ard} {var_mode}] |g − oracle|/max|g| {err:.3e}  dlml {abs(lml - ref_lml) / abs(ref_lml):.2e}")
    assert abs(lml - ref_lml) <= TOL_LML * abs(ref_lml), (lml, ref_lml)
    assert err <= TOL_GRAD, (err, np.argmax(np.abs(g - ref_g)))
    # central differences in log θ = (log amplitude, log noise, log ℓ_1..P) of the engine's LML
    h = 2e-4
    base = dict(amplitude=th["amplitude"], noise=th["noise"], length_scale=np.atleast_1d(th["length_scale"]).astype(float))
    fd = np.empty_like(g)
    for c in range(len(g)):
        vals = []
        for sgn in (1.0, -1.0):
            t = dict(base, length_scale=base["length_scale"].copy())
            if c == 0:
                t["amplitude"] *= np.exp(sgn * h)
            elif c == 1:
                t["noise"] *= np.exp(sgn * h)
            else:
                t["length_scale"][c - 2] *= np.exp(sgn * h)
            f = H.engine({**th, **t}, "f64")
            f.tell(X, y)
            vals.append(f.fit_info()["lml"])
            f.close()
        fd[c] = (vals[0] - vals[1]) / (2 * h)
    fderr = np.abs(fd - g).max() / scale
    print(f"    |g − central differences|/max|g| {fderr:.3e}")
    assert fderr <= TOL_FD, (fderr, np.argmax(np.abs(fd - g)))


def test_lml_batch_at_8192_matches_full_fits_and_lapack(refs):
    """kbo_lml_batch at N = 8192 with G = 4 (the optimizer's batch at that N; the trsv kernel's z takes 64 KB of shared memory):
    three isotropic θ and one ARD θ, each against a full kbo_fit at that θ and against LAPACK (gp_fit)."""
    N, D = 8192, 32
    X, y, _, th = H.history(N, "m32", M=1)
    ls = th["length_scale"]
    thetas = [dict(length_scale=ls, noise=1e-3), dict(length_scale=0.5 * ls, noise=1e-2), dict(length_scale=2.0 * ls, noise=3e-4),
              dict(length_scale=np.linspace(0.6, 1.5, D) * ls, noise=1e-3)]
    e = H.engine(th, "f64")
    got, info = e.lml_batch(X, y, thetas, return_info=True)
    e.close()
    assert np.all(info == 0), info
    for t, g in zip(thetas, got):
        one = H.engine({**th, **t}, "f64")
        one.tell(X, y)
        full = one.fit_info()["lml"]
        one.close()
        lap = O.gp_fit(X, y, kind=th["kind"], length_scale=t["length_scale"], amplitude=th["amplitude"], noise=t["noise"])["lml"]
        print(f"\n[lml_batch N={N} noise={t['noise']}] batch vs fit {abs(g - full) / abs(full):.2e}, vs LAPACK {abs(g - lap) / abs(lap):.2e}")
        assert abs(g - full) <= TOL_LML * abs(full), (t, g, full)
        assert abs(g - lap) <= TOL_LML * abs(lap), (t, g, lap)


# ---- the non-positive-pivot report ---------------------------------------------------------------------------------------------
PIVOTS = (2, 64, 65, 256, 257, 2985)


def _pivot_cases(N):
    return [(N, p) for p in PIVOTS + (N,)]


def _assert_reports(r, where):
    name = f"{where} N={r['N']} p={r['p']}"
    assert r["info"] == r["p"], f"{name}: info {r['info']}"
    assert r["fit_info_rc"] == -3, name
    for call in ("ask", "ask_multi", "predict_mean", "lml_grad"):
        assert r[call] == "not_pd", f"{name}: {call} -> {r[call]}"
    assert r["abi_lml_grad_rc"] == -3, f"{name}: kbo_lml_grad returned {r['abi_lml_grad_rc']}"


@pytest.mark.parametrize("N", [4096, 5800])
def test_non_positive_pivot_is_reported_at_its_index_in_every_schedule(N, tmp_path):
    """oracle.not_pd_at(N, p) fails at exactly pivot p (LAPACK agrees: test_oracle.py).  The default fit, a lazy tensor-core fit,
    and the one-stream schedule must report info == p, and every call that needs the factorisation — ask, ask_multi,
    predict_mean, the LML gradient (also at the C ABI) — must report KBO_ERR_NOT_PD."""
    for var_mode in ("f64", "tc"):
        for r in H.pivots(_pivot_cases(N), var_mode):
            _assert_reports(r, f"v3 {var_mode}")
    for r in _helper({"pivots": _pivot_cases(N), "var_mode": "f64"}, tmp_path / "serial.json", {"KBO_FIT_SERIAL": "1"}):
        _assert_reports(r, "serial")


def test_lml_batch_failing_theta_mid_batch():
    """A θ whose Gram matrix fails at pivot p, in the middle of a batch: −inf and info == p for it, the other θ bit-identical to
    the batch without it."""
    N, p = 4096, 2985
    X, y = O.not_pd_at(N, p)
    e = H.pivot_engine("f64")
    good = [dict(noise=1e-3), dict(noise=1e-2, length_scale=1.5), dict(noise=1e-4, length_scale=np.array([0.8, 1.0, 1.2, 1.4]))]
    got, info = e.lml_batch(X, y, good[:2] + [dict(noise=0.0)] + good[2:], return_info=True)
    ref, rinfo = e.lml_batch(X, y, good, return_info=True)
    e.close()
    assert got[2] == -np.inf and info[2] == p, (got, info)
    assert np.all(rinfo == 0) and np.all(np.isfinite(ref))
    assert np.array_equal(np.delete(got, 2), ref) and np.all(np.delete(info, 2) == 0)


def _same_state(a, b, atol=2e-10):
    for x, z in zip(H.state(a), H.state(b)):
        np.testing.assert_allclose(x.cpu().numpy(), z.cpu().numpy(), rtol=0, atol=atol)
    la, lb = a.fit_info()["lml"], b.fit_info()["lml"]
    assert abs(la - lb) <= 1e-9 * max(1.0, abs(lb)), (la, lb)


def test_append_of_a_duplicate_reports_its_row_and_rebase_drops_it():
    """Appending the exact duplicate of an isolated trial fails at that row (info == row + 1); rebasing to the rows before it
    recovers, with the state, LML and suggestion of a fresh fit."""
    N, p = 4096, 2985
    X, y = O.not_pd_at(N, p)
    Xc = np.random.default_rng(5).random((2000, 4)) * 16.0
    for var_mode in ("f64", "tc"):
        e = H.pivot_engine(var_mode)
        e.tell(X[:p - 1], y[:p - 1])
        assert H.fit_info(e) == (0, 0)
        e.append(X[p - 1], y[p - 1])
        assert H.fit_info(e) == (-3, p), var_mode
        e.rebase(p - 1)
        assert H.fit_info(e) == (0, 0), var_mode
        fresh = H.pivot_engine(var_mode)
        fresh.tell(X[:p - 1], y[:p - 1])
        _same_state(e, fresh)
        be, bf = e.ask(Xc), fresh.ask(Xc)
        assert be.index == bf.index and abs(be.value - bf.value) <= 1e-10 * max(1.0, abs(bf.value)), var_mode
        e.close(); fresh.close()


def test_a_good_fit_after_a_failed_one_on_the_same_handle_is_bit_identical_to_a_fresh_handle():
    """The aborted multi-stream schedule must leave nothing behind: after a failure at p, a good fit on the same handle gives
    bit-identical L, alpha and suggestion to the same fit on a fresh handle."""
    X, y, Xc = O.synthetic(4096, 4096, 32)
    th = dict(kind="matern52", **O.theta_of_record(32))
    for var_mode in ("f64", "tc"):
        for p in (257, 2985):
            Xb, yb = O.not_pd_at(4096, p)
            e = H.engine(th, var_mode)
            e.kernel, e.length_scale, e.noise = "rbf", np.array([1.0]), 0.0
            e.tell(Xb, yb)
            assert H.fit_info(e) == (-3, p)
            e.kernel, e.length_scale, e.noise = th["kind"], np.atleast_1d(th["length_scale"]).astype(float), th["noise"]
            e.tell(X, y)
            f = H.engine(th, var_mode)
            f.tell(X, y)
            be, bf = e.ask(Xc), f.ask(Xc)
            (Le, _, ae), (Lf, _, af) = H.state(e, with_w=False), H.state(f, with_w=False)
            assert torch.equal(torch.tril(Le), torch.tril(Lf)) and torch.equal(ae, af), (var_mode, p)
            assert (be.index, be.value, be.mu, be.std) == (bf.index, bf.value, bf.mu, bf.std), (var_mode, p)
            e.close(); f.close()


@pytest.mark.parametrize("b", [5, 46])
@pytest.mark.parametrize("var_mode", ["f64", "tc"])
def test_rebase_after_a_failed_fit_never_keeps_unfactored_rows(b, var_mode):
    """A fit failing at p = 64·b + 41 stops at the whole 64-block [64·b, 64·b + 64): that block of L and W is never written.
    kbo_fit_rebase(n_keep) then recovers only for n_keep ≤ 64·b — the state, LML and suggestion of a fresh fit of those rows —
    and for n_keep inside the block (64·b + 20, p − 1, p) keeps reporting KBO_ERR_NOT_PD rather than a state built on Gram values."""
    from kubeflow_b200 import _lib as Lb
    N, p = 4096, 64 * b + 41
    X, y = O.not_pd_at(N, p)
    Xc = np.random.default_rng(5).random((2000, 4)) * 16.0
    for n_keep in (64 * b, 64 * b + 20, p - 1, p):
        e = H.pivot_engine(var_mode)
        e.tell(X, y)
        assert H.fit_info(e) == (-3, p)
        e.rebase(n_keep)
        rc, info = H.fit_info(e)
        if n_keep <= 64 * b:
            assert (rc, info) == (0, 0), (n_keep, rc, info)
            fresh = H.pivot_engine(var_mode)
            fresh.tell(X[:n_keep], y[:n_keep])
            _same_state(e, fresh)
            be, bf = e.ask(Xc), fresh.ask(Xc)
            assert be.index == bf.index and abs(be.value - bf.value) <= 1e-10 * max(1.0, abs(bf.value)), n_keep
            fresh.close()
        else:
            assert (rc, info) == (-3, p), (n_keep, rc, info)
            with pytest.raises(Lb.KboNotPositiveDefinite):
                e.ask(Xc)
        e.close()
