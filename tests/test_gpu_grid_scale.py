"""Every acquisition and gp_hedge at the grid sizes the engine serves, against an exhaustive FP64 posterior of the whole grid.

The reference (tests/_posterior_ref.py) is torch's FP64 cholesky / solve_triangular with distances by exact differences: it shares
no code with libkbo and is pinned against scikit-learn and the oracle on the CPU (tests/test_posterior_ref.py).  Each case is one
history and one grid; its reference runs once and serves every check:
  (a) the reference against oracle.gp_fit / gp_predict on 4096 sampled rows and each acquisition's argmax row;
  (b) the FP64 engine's μ, σ and EI / LCB / PI arrays against the reference on EVERY row;
  (c) the default array-free path (auto mode: the tensor-core sweep on a lazy fit with the pruning pass; the FP64 contraction at
      cfg2) for each acquisition on a fresh tell: the reference's first-index argmax, its value to ε, the FP64 engine's value to
      1e-10, decided in FP64.  Gap rule: where the reference's top-1 − top-2 gap is ≤ 2ε, any row within 2ε of the maximum will do;
  (d) gp_hedge (ask_multi ei, lcb, pi): each pick as (c), each equal to its single sweep, the same decisions;
  (e) the grid as three uneven shards with global_offset, max-reduced by (value, −index): what (c) picks;
(f) cfg5's 16,777,216-row grid as eight 2,097,152-row shards on one GPU, EI, against the reference on four of them (the two with
the best picks, two drawn at random); and (g) the FP64 engine's arrays do not depend on its scratch size (many chunks, a ragged
last one, a chunk of more than 2³¹ doubles).  A pick is checked by its value and by its μ and σ: EI at a sharply peaked maximum is
the improvement alone, so σ² scaled by (1 + 1e-6) in both FP64 variance paths moves the EI value by 2e-13 but σ by 1e-7.

Bounds are 4× the worst value measured on one H100 80GB HBM3 (400 W power limit), per case.  Units: y_std for μ, σ, EI and LCB;
1 for PI.  Worst values, each over EI, LCB and PI:
                      (a) reference − oracle   (b) FP64 engine − reference on every row               gap of the reference
                      worst quantity           |dμ|      |dσ|      |d acq|    (row of the acq one)    EI / LCB / PI
  cfg3                4.0e-13 (μ)              7.8e-13   2.4e-14   7.8e-13    (LCB @ 401426)          0.62 / 0.61 / 1.1e-16
  cfg3-raw-y          1.5e-12 (μ, LCB)         1.5e-12   3.5e-14   3.0e-12    (LCB @ 1524)            3.1  / 3.0  / 1.1e-16
  cfg3-ard            6.1e-13 (μ)              1.1e-12   2.5e-14   1.1e-12    (LCB, PI)               0.23 / 0.22 / 0
  n4097-rbf           1.9e-12 (μ, LCB)         2.5e-12   8.1e-14   3.9e-12    (PI @ 287632)           0.80 / 0.79 / 0
  cfg2                2.4e-11 (PI)             2.0e-11   2.1e-13   5.7e-11    (PI @ 787)              0.12 / 0.11 / 1.8e-3
  near-trials-1e-3    5.7e-13 (LCB)            7.6e-13   3.9e-13   1.1e-12    (LCB @ 50386)           0.62 / 0.61 / 1.1e-16
  near-trials-1e-6    3.1e-11 (LCB)            9.3e-13   1.4e-11   2.7e-11    (LCB @ 108940)          0.63 / 0.62 / 2.2e-16
The gaps are raw acquisition values (EI, LCB in units of y, PI unitless); PI saturates at 1 near its maximum, so its pick is held
by the gap rule.  Next to trials (noise 1e-6, σ ≈ 1e-3·y_std) |dσ| is 9.4e-12 on the 4096 exact copies and 1.4e-11 on the 4096
copies moved by 1e-7: the FP64 K* kernel forms r² = ‖a‖² + ‖b‖² − 2a·b, which cancels there, but its absolute error (~1e-15 on
k) moves σ² by ~1e-14, and the two FP64 references (torch and the CPU oracle) differ from each other by as much (1.6e-11).  The
kernel is left as it is.  The default path's pick is the reference's first-index argmax in every case, EI and LCB decided among
1 to 6 survivors of the pruning pass, PI among 350 to 2800 contenders; at the pick its value and μ are the reference's to
≤ 1.1e-12·y_std (cfg2: 9.6e-12), σ to ≤ 5.6e-14·y_std, and the value is the FP64 engine's to ≤ 1.4e-13.  cfg5's pick (row 11,435,952 of 16M) is the reference's with a gap of 0.67.
"""
import dataclasses
import time

import numpy as np
import pytest
import torch

from kubeflow_b200 import workload as W
from oracle import gp_oracle as O
from tests import _grid_cases as G
from tests import _posterior_ref as R

pytestmark = pytest.mark.gpu

ACQS = R.ACQS

# the cases of tests/_grid_cases.py this file runs
SCALE_CASES = ("cfg3", "cfg3-raw-y", "cfg3-ard", "n4097-rbf", "cfg2", "near-trials-1e-3", "near-trials-1e-6")
# (b): bounds on max |μ|, |σ| and |acquisition| of the FP64 engine against the reference, 4× the worst measured (header); the
# acquisition bound is the ε of (c)-(f)
BOUNDS = {"cfg3": (3.2e-12, 9.7e-14, 3.1e-12), "cfg3-raw-y": (6.0e-12, 1.4e-13, 1.2e-11), "cfg3-ard": (4.6e-12, 1.0e-13, 4.6e-12),
          "n4097-rbf": (9.9e-12, 3.3e-13, 1.6e-11), "cfg2": (8.2e-11, 8.5e-13, 2.3e-10), "near-trials-1e-3": (3.1e-12, 1.6e-12, 4.2e-12),
          "near-trials-1e-6": (3.8e-12, 5.6e-11, 1.1e-10)}
BOUNDS["cfg5"] = BOUNDS["cfg3"]
# (a): bound on every quantity of the reference against the CPU oracle, 4× the worst measured
ORACLE_BOUND = {"cfg3": 1.7e-12, "cfg3-raw-y": 6.0e-12, "cfg3-ard": 2.5e-12, "n4097-rbf": 7.5e-12, "cfg2": 9.6e-11, "near-trials-1e-3": 2.3e-12,
                "near-trials-1e-6": 1.3e-10}


@pytest.fixture(scope="module", params=SCALE_CASES)
def case(request):
    """One case's data and its reference; pytest runs every check of a case before the next case is built."""
    d = G.case_data(request.param)
    th = d["theta"]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ref = R.posterior(d["X"], d["y"], d["Xc"], kind=d["kind"], **th, device="cuda")
    torch.cuda.synchronize()
    ref["y_std"] = ref.pop("fit")["y_std"]           # the fit's device tensors go with it
    torch.cuda.empty_cache()
    print(f"\n[{d['name']}] reference over {d['M']} rows in {time.perf_counter() - t0:.1f} s: "
          + " ".join(f"{a} top-1 {ref['top'][a][1]:.6g} @ {ref['top'][a][0]} gap {ref['top'][a][1] - ref['top'][a][2]:.3e}" for a in ACQS))
    d["ref"] = ref
    d["memo"] = {}
    yield d
    d.clear()
    torch.cuda.empty_cache()


def _engine(d, var_mode="auto", acq="ei", **kw):
    from kubeflow_b200.gp import GPEngine
    return GPEngine(0, kernel=d["kind"], acq=acq, var_mode=var_mode, **d["theta"], **kw)


def _scale(d, acq):
    return 1.0 if acq == "pi" else d["ref"]["y_std"]


def _eps(d, acq):
    return BOUNDS[d["name"]][2] * _scale(d, acq)


def _rows(Xc, idx):
    return (Xc[torch.as_tensor(idx, device=Xc.device)].cpu().numpy() if isinstance(Xc, torch.Tensor) else Xc[idx]).astype(np.float64)


def _check_pick(d, acq, b, label):
    """The gap rule: the reference's first-index argmax, or — where its top-1 − top-2 gap is ≤ 2ε — a row within 2ε of the
    maximum; the value within ε of the reference's at the returned row, and μ and σ there within the bounds of (b) (EI at a
    sharply peaked maximum is the improvement alone, whatever σ is)."""
    ref = d["ref"]
    i1, v1, v2 = ref["top"][acq]
    eps = _eps(d, acq)
    a = ref["acq"][acq]
    msg = f"{label}: index {b.index} value {b.value!r}; reference argmax {i1} value {v1!r} gap {v1 - v2:.3e} eps {eps:.1e}"
    assert 0 <= b.index < len(a), msg
    if v1 - v2 > 2 * eps:
        assert b.index == i1, msg
    else:
        assert a[b.index] >= v1 - 2 * eps, msg
    assert abs(b.value - a[b.index]) <= eps, msg + f" reference at the pick {a[b.index]!r}"
    bmu, bsd, _ = BOUNDS[d["name"]]
    dmu, dsd = abs(b.mu - ref["mu"][b.index]), abs(b.std - ref["std"][b.index])
    assert dmu <= bmu * ref["y_std"] and dsd <= bsd * ref["y_std"], msg + f" |dμ| {dmu:.2e} |dσ| {dsd:.2e} at the pick"


def _fp64(d):
    """The FP64 engine's Best and μ, σ, acquisition arrays (host) for each acquisition, one fresh tell per acquisition."""
    if "fp64" not in d["memo"]:
        e = _engine(d, "f64")
        out = {}
        t0 = time.perf_counter()
        for a in ACQS:
            e.acq = a
            e.tell(d["X"], d["y"])
            b, mu, sd, ac = e.ask(d["Xc"], return_arrays=True)
            out[a] = (b, mu.cpu().numpy(), sd.cpu().numpy(), ac.cpu().numpy())
            del mu, sd, ac
        e.close()
        torch.cuda.empty_cache()
        print(f"\n[{d['name']}] FP64 engine, three sweeps with arrays: {time.perf_counter() - t0:.1f} s")
        d["memo"]["fp64"] = out
    return d["memo"]["fp64"]


def _singles(d):
    """The default array-free path, one acquisition at a time on a fresh tell: (Best, (unrefined, contenders, prefix survivors))."""
    if "singles" not in d["memo"]:
        e = _engine(d)
        out = {}
        for a in ACQS:
            e.acq = a
            e.tell(d["X"], d["y"])
            b = e.ask(d["Xc"])
            out[a] = (b, (e.last_unrefined(), e.last_contenders(), e.last_prefix_survivors()))
        e.close()
        d["memo"]["singles"] = out
    return d["memo"]["singles"]


# ---- (a) --------------------------------------------------------------------------------------------------------------------
def test_reference_against_the_cpu_oracle(case):
    d, ref, th = case, case["ref"], case["theta"]
    sample = np.unique(np.concatenate([np.random.default_rng(9).choice(d["M"], 4096, replace=False), [ref["top"][a][0] for a in ACQS]]))
    t0 = time.perf_counter()
    fit = O.gp_fit(d["X"], d["y"], kind=d["kind"], length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    mu, sd = O.gp_predict(fit, _rows(d["Xc"], sample))
    errs = {"mu": np.abs(mu - ref["mu"][sample]).max() / ref["y_std"], "std": np.abs(sd - ref["std"][sample]).max() / ref["y_std"]}
    for a in ACQS:
        oa = O.acquisition(mu, sd, float(np.min(d["y"])), a, th["xi"], th["kappa"])
        errs[a] = np.abs(oa - ref["acq"][a][sample]).max() / _scale(d, a)
    print(f"\n[{d['name']}] (a) reference vs oracle on {len(sample)} rows ({time.perf_counter() - t0:.1f} s): "
          + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert abs(fit["y_std"] - ref["y_std"]) <= 1e-12 * fit["y_std"]     # NumPy and torch sum y in different orders
    for k, v in errs.items():
        assert v <= ORACLE_BOUND[d["name"]], (k, v)


# ---- (b) --------------------------------------------------------------------------------------------------------------------
def test_fp64_engine_arrays_on_every_row(case):
    d, ref = case, case["ref"]
    bmu, bsd, bacq = BOUNDS[d["name"]]
    bad = []
    for a, (b, mu, sd, ac) in _fp64(d).items():
        s = ref["y_std"]
        dm, ds, da = np.abs(mu - ref["mu"]), np.abs(sd - ref["std"]), np.abs(ac - ref["acq"][a])
        im, is_, ia = int(np.argmax(dm)), int(np.argmax(ds)), int(np.argmax(da))
        line = (f"[{d['name']}] (b) {a}: max|dμ| {dm[im] / s:.2e} @ {im}  max|dσ| {ds[is_] / s:.2e} @ {is_} (σ {ref['std'][is_] / s:.2e})  "
                f"max|d acq| {da[ia] / _scale(d, a):.2e} @ {ia}")
        if d["near"] is not None:
            n = len(d["near"]) // 2
            line += "  near rows: " + " ".join(f"{k} {x[rows].max() / s:.2e}" for k, x, rows in
                                               (("dσ copies", ds, d["near"][:n]), ("dσ +1e-7", ds, d["near"][n:])))
        print("\n" + line)
        if dm[im] > bmu * s or ds[is_] > bsd * s or da[ia] > bacq * _scale(d, a):
            bad.append(line)
        if not (b.index == int(np.argmax(ac)) and b.value == ac[b.index]):
            bad.append(f"{a}: Best {b} is not the first maximum of its own array")
    assert not bad, bad


# ---- (c) --------------------------------------------------------------------------------------------------------------------
def test_default_path_picks_the_reference_argmax(case):
    d = case
    fp64 = _fp64(d)
    for a, (b, dec) in _singles(d).items():
        b6 = fp64[a][0]
        i1, v1, v2 = d["ref"]["top"][a]
        ref, s = d["ref"], d["ref"]["y_std"]
        print(f"\n[{d['name']}] (c) {a}: index {b.index} (reference {i1}, gap {v1 - v2:.3e}) |value − reference| "
              f"{abs(b.value - ref['acq'][a][b.index]) / _scale(d, a):.2e} |dμ| {abs(b.mu - ref['mu'][b.index]) / s:.2e} "
              f"|dσ| {abs(b.std - ref['std'][b.index]) / s:.2e}; |value − FP64 engine| {abs(b.value - b6.value):.2e}  "
              f"unrefined {dec[0]} contenders {dec[1]} prefix survivors {dec[2]}")
        _check_pick(d, a, b, f"{d['name']} {a}")
        assert abs(b.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value)), (a, b.value, b6.value)
        assert dec[0] == 0, (a, dec)
        assert (dec[2] != -1) == d["tc"], (a, dec)       # the pruning pass ran where the tensor-core path is taken


# ---- (d) --------------------------------------------------------------------------------------------------------------------
def test_gp_hedge_picks_what_each_single_sweep_picks(case):
    d = case
    singles = _singles(d)
    e = _engine(d)
    e.tell(d["X"], d["y"])
    multi = e.ask_multi(d["Xc"], list(ACQS))
    dec = e.last_decisions()
    e.close()
    print(f"\n[{d['name']}] (d) ask_multi decisions {dec}, single sweeps {[singles[a][1] for a in ACQS]}")
    for k, a in enumerate(ACQS):
        b, s = multi[k], singles[a][0]
        _check_pick(d, a, b, f"{d['name']} gp_hedge {a}")
        assert b.index == s.index, (a, b.index, s.index)
        for fld in ("value", "mu", "std"):
            x, y = getattr(b, fld), getattr(s, fld)
            assert abs(x - y) <= 1e-12 * max(1.0, abs(y)), (a, fld, x, y)
        single = singles[a][1]
        # the FP64 contraction refines nothing: kbo_last_contenders keeps what an earlier sweep left there
        assert dec[k] == (single if d["tc"] else (single[0], dec[k][1], single[2])), (a, dec[k], single)


# ---- (e) --------------------------------------------------------------------------------------------------------------------
def test_three_uneven_shards_reduce_to_the_single_sweep(case):
    d = case
    M = d["M"]
    cuts = [0, int(0.23 * M) + 5, int(0.61 * M) + 77, M]
    singles = _singles(d)
    e = _engine(d)
    for a in ACQS:
        e.acq = a
        parts = []
        for s0, s1 in zip(cuts[:-1], cuts[1:]):
            e.tell(d["X"], d["y"])                     # every rank holds a fresh fit of its own
            parts.append(e.ask(d["Xc"][s0:s1], global_offset=s0))
        win = max(parts, key=lambda b: (b.value, -b.index))
        s = singles[a][0]
        print(f"\n[{d['name']}] (e) {a}: shard picks {[(p.index, p.value) for p in parts]} -> {win.index}")
        _check_pick(d, a, win, f"{d['name']} shards {a}")
        assert win.index == s.index and abs(win.value - s.value) <= 1e-12 * max(1.0, abs(s.value)), (a, win, s)
    e.close()


# ---- (f) --------------------------------------------------------------------------------------------------------------------
def test_cfg5_grid_of_16m_rows_as_eight_shards():
    """cfg5's grid (16,777,216 rows, D = 32, the cfg3 history) swept as the eight 2,097,152-row shards its ranks own, on one GPU,
    EI, each shard on a fresh fit.  The reference over all 16M rows takes 2.5 minutes on an H100, so it runs on four shards: the two
    whose picks (each decided in FP64) are the best, and two others drawn at random.  The max-reduced pick must be the reference's
    argmax over those shards by the gap rule, and every checked shard's own pick the reference's argmax of that shard.  This is
    the decision at cfg5's per-rank shape; test_gpu_spmd.py covers the NCCL exchange."""
    N, D, Mr, R8 = 8192, 32, 2_097_152, 8
    X, y, _ = O.synthetic(N, 1, D)
    th = O.theta_of_record(D)
    t0 = time.perf_counter()
    e = _engine(dict(kind="matern52", theta=th))
    parts, decs = [], []
    for r in range(R8):
        xc = torch.tensor(W.candidates(Mr, D, offset=r * Mr), device="cuda")
        e.tell(X, y)
        parts.append(e.ask(xc, global_offset=r * Mr))
        decs.append((e.last_unrefined(), e.last_contenders(), e.last_prefix_survivors()))
        del xc
    e.close()
    torch.cuda.empty_cache()
    order = sorted(range(R8), key=lambda r: (parts[r].value, -parts[r].index), reverse=True)
    checked = sorted(order[:2] + [int(r) for r in np.random.default_rng(5).choice(order[2:], 2, replace=False)])
    f = R.fit(X, y, kind="matern52", length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"], device="cuda")
    a_all, mu_all, sd_all = np.full(R8 * Mr, -np.inf), np.full(R8 * Mr, np.nan), np.full(R8 * Mr, np.nan)
    for r in checked:
        xc = torch.tensor(W.candidates(Mr, D, offset=r * Mr), device="cuda")
        rows = slice(r * Mr, (r + 1) * Mr)
        mu_all[rows], sd_all[rows] = R.predict(f, xc)
        del xc
        a_all[rows] = O.acquisition(mu_all[rows], sd_all[rows], f["y_opt"], "ei", th["xi"], th["kappa"])
    y_std = f["y_std"]
    del f
    torch.cuda.empty_cache()
    win = max(parts, key=lambda b: (b.value, -b.index))
    d = dict(name="cfg5", ref=dict(acq={"ei": a_all}, top={"ei": R.top2(a_all)}, mu=mu_all, std=sd_all, y_std=y_std))
    i1, v1, v2 = d["ref"]["top"]["ei"]
    print(f"\n[cfg5] {time.perf_counter() - t0:.1f} s, reference on shards {checked}: pick {win.index} value {win.value:.10f}; reference "
          f"{i1} {v1:.10f} gap {v1 - v2:.3e}; per shard (pick, value) {[(p.index, round(p.value, 6)) for p in parts]}, "
          f"(unrefined, contenders, prefix survivors) {decs}")
    _check_pick(d, "ei", win, "cfg5")
    for r in checked:
        rows = slice(r * Mr, (r + 1) * Mr)
        d_r = dict(name="cfg5", ref=dict(acq={"ei": a_all[rows]}, top={"ei": R.top2(a_all[rows])}, mu=mu_all[rows], std=sd_all[rows],
                                         y_std=y_std))
        _check_pick(d_r, "ei", dataclasses.replace(parts[r], index=parts[r].index - r * Mr), f"cfg5 shard {r}")
    assert all(u == 0 for u, _, _ in decs), decs


# ---- (g) --------------------------------------------------------------------------------------------------------------------
def _f64_arrays(X, y, xc, th, **kw):
    from kubeflow_b200.gp import GPEngine
    e = GPEngine(0, kernel="matern52", acq="ei", var_mode="f64", **th, **kw)
    e.tell(X, y)
    b, mu, sd, a = e.ask(xc, return_arrays=True)
    out = (b, mu.cpu().numpy(), sd.cpu().numpy(), a.cpu().numpy())
    e.close()
    del mu, sd, a
    torch.cuda.empty_cache()
    return out


def test_fp64_engine_arrays_do_not_depend_on_the_scratch_size():
    """cfg3's history and the first 1,048,539 rows of its grid through the FP64 engine at the default scratch (4 GiB: 65,536-row
    chunks), at 256 MiB (4096-row chunks, the last one 4059 rows; each so small that the K* kernel splits its trial tiles, so the
    mean may differ by summation order) and at 17 GiB (278,528-row chunks: more than 2³¹ doubles of K* in one chunk — bit for bit
    the default's, no chunk being split)."""
    N, D, M = 8192, 32, 1_048_539
    X, y, _ = O.synthetic(N, 1, D)
    th = O.theta_of_record(D)
    xc = torch.tensor(W.candidates(M, D), device="cuda")
    b0, mu0, sd0, a0 = _f64_arrays(X, y, xc, th)
    b1, mu1, sd1, a1 = _f64_arrays(X, y, xc, th, scratch_limit=256 << 20)
    dmu = np.abs(mu1 - mu0).max()
    print(f"\n(g) 256 MiB: max|dμ| {dmu:.2e} max|dσ| {np.abs(sd1 - sd0).max():.2e} max|d acq| {np.abs(a1 - a0).max():.2e}")
    tol_mu = 1e-12 * max(1.0, float(np.abs(mu0).max()))
    assert dmu <= tol_mu
    np.testing.assert_allclose(sd1, sd0, rtol=1e-12, atol=0)
    np.testing.assert_allclose(a1, a0, rtol=1e-12, atol=tol_mu)
    assert b1.index == b0.index and abs(b1.value - b0.value) <= 1e-12 * max(1.0, abs(b0.value))
    free, total = torch.cuda.mem_get_info()
    need = 24 << 30
    if free < need:
        pytest.skip(f"17 GiB scratch: {free / 2**30:.1f} GiB of {total / 2**30:.1f} GiB free, the case needs {need / 2**30:.0f} GiB")
    b2, mu2, sd2, a2 = _f64_arrays(X, y, xc, th, scratch_limit=17 << 30)
    print(f"(g) 17 GiB: max|dμ| {np.abs(mu2 - mu0).max():.2e} max|dσ| {np.abs(sd2 - sd0).max():.2e} max|d acq| {np.abs(a2 - a0).max():.2e}")
    assert np.array_equal(mu2, mu0) and np.array_equal(sd2, sd0) and np.array_equal(a2, a0)
    assert (b2.index, b2.value) == (b0.index, b0.value)
