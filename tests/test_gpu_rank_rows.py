"""The tensor-core ranking arithmetic row by row against the FP64 posterior, and every pruning bound on every row.

An array-free suggestion is a branch-and-bound (DESIGN.md §1): the tensor-core K* kernel gives a mean μ̃, the wgmma kernel a
one-product variance σ̃² (over a prefix of the trial tiles in the pruning pass, over all of them in the ranking pass), and rows are
pruned against E = 8·max|σ̃² − σ²| + 1e-6 and Eμ = 8·max|μ̃ − μ| + 1e-7 measured on the stratified calibration rows.  A row pruned
wrongly is never seen again, so the picks of test_gpu_grid_scale.py prove only that the argmax row survived.  Here the reference
(tests/_posterior_ref.predict_normalised: μ_n, σ²_n and the exact prefix variance σ²_P, P = the pruning pass's trials) checks:
  (a) the tensor-core K* plane on 4096 sampled rows and each acquisition's reference argmax: within 0.51 fp16 ulp + 2e-6 of the
      FP64 kernel value, zero in the padding columns;
  (b) EVERY row (kbo_debug_rank_rows, the grid in 131,072-row slices) against the E and Eμ each stage of a sweep recorded
      (kbo_debug_record_stages): |μ̃ − μ_n| ≤ Eμ; σ̃²_prefix + E ≥ σ²_P ≥ σ²_n in the lazy-fit and the full-fit pruning pass;
      |σ̃²_full − σ²_n| ≤ E for the ranking pass's interval test; and the three-product variance (tc arrays) to 4× its measured
      error, below the 2e-4 window its redo relies on;
  (c) in every stage of every sweep, EI, LCB and PI, default / lazy_inverse=False / rank_prefix=0 / tc_fast=False: the survivor
      threshold ≤ the reference maximum (normalised units), and every row within ε of the maximum among the survivors;
  (d) each of those sweeps and gp_hedge pick the reference's first-index argmax by the gap rule of test_gpu_grid_scale.py, decided
      in FP64 (last_unrefined 0);
  (e) a row's μ̃, σ̃²_prefix and σ̃²_full do not depend on its position: the grid reversed and rolled by 12,345 rows, in ragged
      slices, gives the same values bit for bit — what makes slicing (b) and calibrating on a sample legitimate.

Measured on one H100 80GB HBM3 at a 400 W power limit.  Worst row's share of its bound, over every row: |μ̃ − μ_n|/Eμ (the same
μ̃ in every stage); (σ²_P − σ̃²_P)/E in the lazy-fit and in the full-fit pruning pass; |σ̃² − σ²_n|/E in the interval test; and
the three-product variance's |σ²₃ − σ²_n|/amplitude.  No worst row is a calibration row.
                     Eμ      lazy E   full-fit E   interval E   three products
  cfg3               0.162   0.151    0.074        0.155        3.7e-6
  cfg3-raw-y         0.165   0.139    0.068        0.141        3.6e-6
  n4097-rbf          0.145   0.176    0.073        0.139        4.6e-6
  d128               0.136   0.143    0.090        0.146        2.5e-6
  near-trials-1e-6   0.157   0.154    0.075        0.141        3.8e-6
  amp-1e3            0.155   0.138    0.072        0.149        3.7e-6
  ls5-noise-1e-6     0.153   0.130    0.005        0.127        1.5e-5
  converged-d4       0.195   0.130    0.026        0.132        2.2e-5
Survivors of each stage on the default path (lazy-fit pruning → full-fit pruning → interval test of the pruning survivors, or
→ interval test over the grid → three-product window), and last_unrefined:
                     EI                               LCB                               PI
  cfg3               1                                1                                 6109 → 6109 → 352
  cfg3-raw-y         1                                1                                 6266 → 6266 → 367
  n4097-rbf          1                                1                                 7207 → 7207 → 3086
  d128               27156 → 248 → 1                  61981 → 404 → 1                   1
  near-trials-1e-6   1                                1                                 6061 → 6061 → 354
  amp-1e3            667513 → 49067 → grid 1          all → 177422 → grid 13            6101 → 6101 → 1
  ls5-noise-1e-6     1                                5                                 14645 → 14645 → 14645 → grid all → window 5701 (2)
  converged-d4       all → all → grid all → window 13 (1)   474987 → 775720 → grid 592643 → window 1   all → all → grid all → window 47 (1)
The other configurations decide at their first stage that fits (lazy_inverse=False at the full-fit pruning pass, rank_prefix=0
at the interval test, tc_fast=False in the window), with the same outcome.  gp_hedge's stages are each single sweep's.
"""
import time

import numpy as np
import pytest
import torch

from tests import _grid_cases as G
from tests import _posterior_ref as R

pytestmark = pytest.mark.gpu

ACQS = R.ACQS
RANK_CASES = ("cfg3", "cfg3-raw-y", "n4097-rbf", "d128", "near-trials-1e-6", "amp-1e3", "ls5-noise-1e-6", "converged-d4")
CONFIGS = {"default": {}, "full-fit": dict(lazy_inverse=False), "no-prefix": dict(rank_prefix=0), "three-product": dict(tc_fast=False)}
# (d) ε of the gap rule (units of y_std; 1 for PI): the bound on the FP64 decision's value against the reference.  The cases
# test_gpu_grid_scale.py also runs take its bound; the others 4× the worst |value − reference| measured here over every
# configuration and acquisition
EPS = {"cfg3": 3.1e-12, "cfg3-raw-y": 1.2e-11, "n4097-rbf": 1.6e-11, "near-trials-1e-6": 1.1e-10,
       "d128": 2.8e-13, "amp-1e3": 1.1e-12, "ls5-noise-1e-6": 7.9e-10, "converged-d4": 4.8e-12}
# (b) the three-product variance (tc arrays) against σ²_n, relative to the amplitude: 4× the worst measured per case
VAR3_BOUND = {"cfg3": 1.5e-5, "cfg3-raw-y": 1.5e-5, "n4097-rbf": 1.9e-5, "d128": 1.1e-5, "near-trials-1e-6": 1.6e-5, "amp-1e3": 1.5e-5,
              "ls5-noise-1e-6": 6.0e-5, "converged-d4": 8.8e-5}
# Where the three-product window cannot hold every row that could be the maximum, the sweep says so (last_unrefined) and the
# test asserts the documented outcome and what still holds: the pick is the reference's first-index argmax itself.
#   converged-d4, EI and PI: a late-stage history on few hyperparameters has a flat landscape — maxima of 2.9e-10·y_std and
#     1.7e-8, below every bound of the pruning passes — so every row survives them, and more than 4096 lie within the window,
#     which narrows until 4096 fit (1): the FP64 decision is taken among the best 4096 by fp32 value.
#   ls5-noise-1e-6, PI: PI is exactly 1 in FP64 and in fp32 on more than 4096 rows (2): the pick is the lowest index among the
#     fp32 ties, which is the lowest index among the FP64 ones.
NARROWED = {("converged-d4", "ei"): 1, ("converged-d4", "pi"): 1, ("ls5-noise-1e-6", "pi"): 2}

def _pairs(N):
    """(tile pairs of the pruning pass, its trials P): an eighth of the pairs of 256-trial tiles, as sweep.cu picks them."""
    npad = (N + 255) // 256 * 256
    n_pairs = (npad // 256 + 1) // 2
    p1 = (n_pairs + 7) // 8
    return p1, p1 * 512


def _xc_cuda(d):
    xc = d["Xc"]
    return xc if isinstance(xc, torch.Tensor) else torch.as_tensor(xc, device="cuda")


@pytest.fixture(scope="module", params=RANK_CASES)
def case(request):
    d = G.case_data(request.param)
    th = d["theta"]
    N = d["X"].shape[0]
    p1, P = _pairs(N)
    t0 = time.perf_counter()
    f = R.fit(d["X"], d["y"], kind=d["kind"], length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"], device="cuda")
    ref = R.predict_normalised(f, d["Xc"], prefixes=(P,))
    ys, ym = f["y_std"], f["y_mean"]
    mu = ys * ref["mu_n"] + ym
    std = np.sqrt(np.maximum(ref["var_n"], 0.0)) * ys
    ref["acq"], ref["top"] = R.acquisitions(mu, std, f["y_opt"], xi=th["xi"], kappa=th["kappa"])
    ref.update(mu=mu, std=std, y_std=ys, y_mean=ym, P=P, p1=p1)
    del f
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    print(f"\n[{d['name']}] reference over {d['M']} rows in {time.perf_counter() - t0:.1f} s (P = {P}): "
          + " ".join(f"{a} top-1 {ref['top'][a][1]:.6g} @ {ref['top'][a][0]} gap {ref['top'][a][1] - ref['top'][a][2]:.3e}" for a in ACQS))
    d.update(ref=ref, memo={})
    yield d
    d.clear()
    torch.cuda.empty_cache()


def _engine(d, acq="ei", var_mode="auto", **kw):
    from kubeflow_b200.gp import GPEngine
    return GPEngine(0, kernel=d["kind"], acq=acq, var_mode=var_mode, **d["theta"], **kw)


def _norm(d, acq, v):
    """A raw acquisition value in the sweep's normalised units (acq_value_f32 in sweep.cu)."""
    ref = d["ref"]
    return v if acq == "pi" else (v + ref["y_mean"]) / ref["y_std"] if acq == "lcb" else v / ref["y_std"]


def _rows(d):
    """The hook's per-row values of the whole grid, each from the fit the stage prunes with: μ̃ and the prefix σ̃² of a lazy fit
    (the lazy-fit pruning pass: W's leading rows only, its fp16 planes scaled by their own maximum), the prefix σ̃² of a full fit
    (lazy_inverse=False: the full-fit pruning pass) and the full σ̃² (the interval test)."""
    if "rows" not in d["memo"]:
        xc = _xc_cuda(d)
        e = _engine(d)
        e.tell(d["X"], d["y"])
        mu_p, var_p = e.rank_rows(xc, d["ref"]["p1"])
        e.close()
        e = _engine(d, lazy_inverse=False)
        e.tell(d["X"], d["y"])
        mu_q, var_q = e.rank_rows(xc, d["ref"]["p1"])
        mu_f, var_f = e.rank_rows(xc, -1)
        e.close()
        d["memo"]["rows"] = {k: v.cpu().numpy() for k, v in dict(mu_p=mu_p, var_p=var_p, mu_q=mu_q, var_q=var_q, mu_f=mu_f, var_f=var_f).items()}
        del mu_p, var_p, mu_q, var_q, mu_f, var_f
        torch.cuda.empty_cache()
    return d["memo"]["rows"]


def _sweeps(d):
    """Each configuration's sweep per acquisition on a fresh tell, recording its stages: {config: {acq: (Best, unrefined, stages)}},
    plus gp_hedge on the default configuration."""
    if "sweeps" not in d["memo"]:
        out = {}
        xc = _xc_cuda(d)
        for name, kw in CONFIGS.items():
            e = _engine(d, **kw).record_stages()
            out[name] = {}
            for a in ACQS:
                e.acq = a
                e.tell(d["X"], d["y"])
                b = e.ask(xc)
                out[name][a] = (b, e.last_unrefined(), [s for s in e.stages() if s["acq"] == a])
            if name == "default":
                e.tell(d["X"], d["y"])
                multi = e.ask_multi(xc, list(ACQS))
                out["gp_hedge"] = {a: (multi[k], e.last_decisions()[k][0], [s for s in e.stages() if s["acq"] == a]) for k, a in enumerate(ACQS)}
            e.close()
        d["memo"]["sweeps"] = out
    return d["memo"]["sweeps"]


def _stage(d, config, stage):
    """The record of a stage of `config`'s EI sweep (its E and Eμ: every acquisition shares the calibration)."""
    for s in _sweeps(d)[config]["ei"][2]:
        if s["stage"] == stage:
            return s
    raise AssertionError(f"{d['name']}: the {config} sweep ran no {stage} stage: {[s['stage'] for s in _sweeps(d)[config]['ei'][2]]}")


def _worst(d, err, bound, label):
    """Worst row of err/bound, as a message naming the row and whether it is a calibration row."""
    ratio = err / bound
    i = int(np.argmax(ratio))
    M = d["M"]
    n = min(M, torch.cuda.get_device_properties(0).multi_processor_count * 64)     # calibration_rows: row k·M/n, k < n
    is_cal = bool(np.any((np.arange(n, dtype=np.int64) * M) // n == i))
    return i, float(ratio[i]), f"{label}: worst row {i} at {ratio[i]:.3f} of the bound ({err[i]:.3e} vs {bound:.3e}), calibration row: {is_cal}"


# ---- (a) --------------------------------------------------------------------------------------------------------------------
def test_kstar_plane_at_production_shapes(case):
    d, ref = case, case["ref"]
    th = d["theta"]
    N = d["X"].shape[0]
    sample = np.unique(np.concatenate([np.random.default_rng(3).choice(d["M"], 4096, replace=False), [ref["top"][a][0] for a in ACQS]]))
    xc = _xc_cuda(d)[torch.as_tensor(sample, device="cuda")]
    e = _engine(d)
    e.tell(d["X"], d["y"])
    _, plane = e.kstar_pass(xc)
    e.close()
    plane = plane[:len(sample)].float()
    ls = torch.as_tensor(np.atleast_1d(th["length_scale"]), device="cuda", dtype=torch.float64)
    Xs = torch.as_tensor(d["X"], device="cuda") / ls
    Kref = R.kernel(xc.double() / ls, Xs, d["kind"], th["amplitude"], 1 << 30)
    ulp = torch.clamp(Kref.abs(), min=2.0 ** -14) * 2.0 ** -10
    excess = ((plane[:, :N].double() - Kref).abs() - (0.51 * ulp + 2e-6)).max().item()
    pad = plane[:, N:].abs().max().item() if plane.shape[1] > N else 0.0
    print(f"\n[{d['name']}] (a) K* plane on {len(sample)} rows: worst |plane − K| − (0.51 ulp + 2e-6) = {excess:.3e}, padding max {pad}")
    assert excess <= 0.0 and pad == 0.0


# ---- (b) --------------------------------------------------------------------------------------------------------------------
def test_every_row_within_the_bounds_each_stage_prunes_with(case):
    d, ref = case, case["ref"]
    rows = _rows(d)
    mu_n, var_n, var_P = ref["mu_n"], ref["var_n"], ref["var_p"][ref["P"]]
    lines, bad = [], []
    # the same K* kernel gives the mean in every pass and either fit; only the stored columns differ
    assert np.array_equal(rows["mu_p"], rows["mu_f"]) and np.array_equal(rows["mu_q"], rows["mu_f"])
    dmu = np.abs(rows["mu_p"].astype(np.float64) - mu_n)
    # σ²_P is an upper bound on σ²_n (exact arithmetic: every V_j² ≥ 0); its FP64 rounding is far below 1e-12
    assert np.all(var_P >= var_n - 1e-12 * np.maximum(1.0, np.abs(var_n)))
    checks = []
    for config, stage, key in (("default", "lazy-prune", "var_p"), ("full-fit", "prune", "var_q")):
        s = _stage(d, config, stage)
        checks.append((f"{stage} |μ̃ − μ_n|", dmu, s["E_mu"]))
        checks.append((f"{stage} σ²_P − σ̃²_P", var_P - rows[key].astype(np.float64), s["E"]))   # above E: the prefix bound fails
        dv = np.abs(rows[key].astype(np.float64) - var_P)
        lines.append(f"{stage}: E {s['E']:.3e} (raw {s['dvar_raw']:.3e}) Eμ {s['E_mu']:.3e} (raw {s['dmu_raw']:.3e}) cal {s['cal_n']}; "
                     f"max|σ̃²_P − σ²_P| {dv.max():.3e} = {dv.max() / s['E']:.3f} E, max|dμ| {dmu.max():.3e} = {dmu.max() / s['E_mu']:.3f} Eμ")
    s = _stage(d, "no-prefix", "interval")
    dvf = np.abs(rows["var_f"].astype(np.float64) - var_n)
    checks.append(("interval |μ̃ − μ_n|", dmu, s["E_mu"]))
    checks.append(("interval |σ̃² − σ²_n|", dvf, s["E"]))
    lines.append(f"interval: E {s['E']:.3e} (raw {s['dvar_raw']:.3e}) Eμ {s['E_mu']:.3e} (raw {s['dmu_raw']:.3e}); "
                 f"max|σ̃² − σ²_n| {dvf.max():.3e} = {dvf.max() / s['E']:.3f} E, max|dμ| {dmu.max() / s['E_mu']:.3f} Eμ")
    for label, err, bound in checks:
        i, ratio, msg = _worst(d, err, bound, label)
        lines.append(msg)
        if not ratio <= 1.0:
            bad.append(msg)
    print(f"\n[{d['name']}] (b) " + "\n    ".join(lines))
    assert not bad, bad


def test_three_product_variance_on_every_row(case):
    d, ref = case, case["ref"]
    e = _engine(d, var_mode="tc")
    e.tell(d["X"], d["y"])
    _, mu, sd, _ = e.ask(_xc_cuda(d), return_arrays=True)
    e.close()
    ys = ref["y_std"]
    var3 = (sd.cpu().numpy() / ys) ** 2
    mu3 = (mu.cpu().numpy() - ref["y_mean"]) / ys
    del mu, sd
    torch.cuda.empty_cache()
    amp = d["theta"]["amplitude"]
    dv = np.abs(var3 - np.maximum(ref["var_n"], 0.0)) / amp
    dm = np.abs(mu3 - ref["mu_n"])
    dsd = np.abs(np.sqrt(var3) - np.sqrt(np.maximum(ref["var_n"], 0.0)))
    i, ratio, msg = _worst(d, dv, VAR3_BOUND[d["name"]], "three-product |σ²₃ − σ²_n| / amplitude")
    print(f"\n[{d['name']}] (b) three products: {msg}; max|μ − μ_n| {dm.max():.3e}, max|σ − σ_n| {dsd.max():.3e} (normalised)")
    assert ratio <= 1.0, msg


# ---- (c) and (d) ------------------------------------------------------------------------------------------------------------
def _near_max_rows(d, acq):
    a = d["ref"]["acq"][acq]
    scale = 1.0 if acq == "pi" else d["ref"]["y_std"]
    return np.flatnonzero(a >= a.max() - EPS[d["name"]] * scale)


CAPS = {"lazy-prune": 16384, "prune": 16384, "prune-interval": 4096, "interval": 4096, "window": 4096}


@pytest.mark.parametrize("config", list(CONFIGS) + ["gp_hedge"])
def test_stages_keep_the_maximum_and_the_pick_is_the_reference_argmax(case, config):
    d, ref = case, case["ref"]
    bad, lines = [], []
    for a in ACQS:
        b, unrefined, stages = _sweeps(d)[config][a]
        vmax = _norm(d, a, ref["top"][a][1])
        near = _near_max_rows(d, a)
        narrowed = (d["name"], a) in NARROWED
        for s in stages:
            if not (s["thr"] <= vmax or np.isnan(s["lb"])):
                bad.append(f"{a} {s['stage']}: threshold {s['thr']!r} above the reference maximum {vmax!r} (lower bound {s['lb']!r})")
            complete = s["n"] <= CAPS[s["stage"]] and not (narrowed and s["stage"] == "window")
            missing = np.setdiff1d(near, s["survivors"]) if complete else np.array([], dtype=np.int64)
            if missing.size:
                bad.append(f"{a} {s['stage']}: {missing.size} of the {near.size} rows within ε of the maximum pruned, e.g. {missing[:5]}")
        lines.append(f"{a}: |value − reference| {abs(b.value - ref['acq'][a][b.index]) / (1.0 if a == 'pi' else ref['y_std']) if 0 <= b.index < d['M'] else np.nan:.2e} " + ", ".join(f"{s['stage']} {s['n']}" + (f" (lb {s['lb'] - vmax:+.2e})" if s['lb'] == s['lb'] else "") for s in stages)
                     + f"; pick {b.index} unrefined {unrefined}")
        i1, v1, v2 = ref["top"][a]
        eps = EPS[d["name"]] * (1.0 if a == "pi" else ref["y_std"])
        if v1 - v2 > 2 * eps:
            ok = b.index == i1
        else:
            ok = 0 <= b.index < d["M"] and ref["acq"][a][b.index] >= v1 - 2 * eps
        if not ok or abs(b.value - ref["acq"][a][b.index if 0 <= b.index < d["M"] else i1]) > eps:
            bad.append(f"{a}: pick {b.index} value {b.value!r}; reference argmax {i1} value {v1!r} gap {v1 - v2:.3e} eps {eps:.1e}")
        if narrowed:
            if not (unrefined == NARROWED[d["name"], a] and b.index == i1):
                bad.append(f"{a}: narrowed window: last_unrefined {unrefined} (expected {NARROWED[d['name'], a]}), pick {b.index}, "
                           f"reference argmax {i1}")
        elif unrefined != 0:
            bad.append(f"{a}: last_unrefined {unrefined}")
    print(f"\n[{d['name']}] (c, d) {config}: " + "; ".join(lines))
    assert not bad, bad


# ---- (e) --------------------------------------------------------------------------------------------------------------------
def test_rows_do_not_depend_on_their_position(case):
    """On one lazy fit: the prefix pass over the grid in its own order (131,072-row slices), reversed (77,777-row slices) and
    rolled (50,001-row slices), then — W completed — the full pass in the same three ways.  Every permuted value is the original's
    bit for bit, and the original-order values are those of _rows, computed on other engines of the same fit.  (The prefix passes
    go first: completing W rescales its fp16 planes to the maximum of all of W, which moves the prefix values of some rows by an
    fp32 rounding — a different fit state, not a different position.)"""
    d = case
    rows = _rows(d)
    xc = _xc_cuda(d)
    M = d["M"]
    e = _engine(d)
    e.tell(d["X"], d["y"])
    orders = (("original", np.arange(M), 131_072), ("reversed", np.arange(M)[::-1].copy(), 77_777), ("rolled", np.roll(np.arange(M), 12_345), 50_001))
    bad = []
    for pairs, keys in ((d["ref"]["p1"], ("mu_p", "var_p")), (-1, ("mu_f", "var_f"))):
        for label, perm, slice_rows in orders:
            xp = xc[torch.as_tensor(perm, device="cuda")]
            vals = e.rank_rows(xp, pairs, slice_rows=slice_rows)
            del xp
            for k, v in zip(keys, vals):
                v = v.cpu().numpy()
                diff = v != rows[k][perm]
                if diff.any():
                    w = np.flatnonzero(diff)
                    bad.append(f"{label} {k}: {w.size} rows differ (first at position {w[0]}), max |d| {np.abs(v[w] - rows[k][perm][w]).max():.3e}")
    e.close()
    torch.cuda.empty_cache()
    print(f"\n[{d['name']}] (e) " + ("; ".join(bad) if bad else "bit for bit"))
    assert not bad, bad
