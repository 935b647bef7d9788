"""The tensor-core suggestion path off the operating point of record: raw y scales (a Katib metric in µs, or a negated
throughput, has |y_mean| in the thousands and y_std of a few units), the θ range the service accepts and the θ search
visits, adversarial near-ties at the calibration rows, and the FP64 engine itself against a long-double restatement where
the FP64 oracle stops being a reference.

Every tensor-core variant of the array-free sweep — pruning pass on a lazy fit (the default), no pruning pass, an eager
fit, three products with the FP64 refinement window — must return the FP64 engine's suggestion: same index, value to
1e-10 relative, decided in FP64 (last_unrefined() == 0)."""
import functools

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

N, M, D = 2048, 30000, 8
KIND = "matern52"
VARIANTS = {"tc": {}, "tc-noprefix": dict(rank_prefix=0), "tc-eager": dict(lazy_inverse=False), "tc-three": dict(tc_fast=False)}


@functools.lru_cache(maxsize=None)
def _data():
    return O.synthetic(N, M, D)


def _engines(acq, normalize_y=True, **theta):
    from kubeflow_b200.gp import GPEngine
    kw = dict(kernel=KIND, acq=acq, normalize_y=normalize_y, **{**O.theta_of_record(D), **theta})
    engs = {name: GPEngine(0, var_mode="tc", **kw, **over) for name, over in VARIANTS.items()}
    engs["f64"] = GPEngine(0, var_mode="f64", **kw)
    return engs


def _close(engs):
    for e in engs.values():
        e.close()


def _check_same(name, e, b, b6, label, rtol=1e-10):
    """The FP64 engine's suggestion, decided in FP64.  One exception, stated in DESIGN.md §1: an EI / PI landscape whose maximum
    is below 1e-30·y_std (no candidate with a measurable improvement — all zero in fp32) may be decided among fp32 ties
    (last_unrefined 1 or 2); the value returned is then still the FP64 maximum to that absolute accuracy."""
    y_std = e.fit_info()["y_std"] if e.normalize_y else 1.0
    msg = (f"{label} [{name}]: index {b.index} value {b.value!r} unrefined {e.last_unrefined()} contenders {e.last_contenders()} "
           f"prefix survivors {e.last_prefix_survivors()}; f64 index {b6.index} value {b6.value!r} (d = {b.value - b6.value:.3e})")
    if e.acq != "lcb" and 0.0 <= b6.value < 1e-30 * y_std:
        assert abs(b.value - b6.value) <= 1e-30 * y_std, msg
        return
    assert (b.index, e.last_unrefined()) == (b6.index, 0) and abs(b.value - b6.value) <= rtol * max(1.0, abs(b6.value)), msg


def _same_decision(engs, X, y, Xc, label):
    """tell + array-free ask on every engine; every tensor-core variant must return the FP64 engine's suggestion."""
    for e in engs.values():
        e.tell(X, y)
    b6 = engs["f64"].ask(Xc)
    for name in VARIANTS:
        _check_same(name, engs[name], engs[name].ask(Xc), b6, label)
    return b6


# ---- (a) raw y scales -------------------------------------------------------------------------------------------------
Y_SCALES = [(0.0, 1.0), (1e3, 1.0), (2e4, 5.0), (-1e5, 2.0), (0.0, 1e-3), (5e5, 1e3)]


@pytest.mark.parametrize("acq", ["ei", "lcb", "pi"])
def test_y_scale_normalized(acq):
    """y = c + s·y₀ with normalize_y: the normalised posterior is the same for every (c, s); the acquisition is evaluated at
    the raw scale, where an fp32 μ = y_mean + y_std·μ_n rounds at the scale of y_mean."""
    X, y0, Xc = _data()
    engs = _engines(acq)
    for c, s in Y_SCALES:
        _same_decision(engs, X, c + s * y0, Xc, f"{acq} c={c:g} s={s:g}")
        # the per-candidate arrays of the tensor-core sweep carry the normalised posterior's error times y_std, not fp32 rounding
        # at the scale of y_mean
        _, mu6, _, a6 = engs["f64"].ask(Xc, return_arrays=True)
        _, mut, _, at = engs["tc"].ask(Xc, return_arrays=True)
        dm, da = float((mut - mu6).abs().max()), float((at - a6).abs().max())
        # PI = Φ((c_n − μ_n)/σ_n) amplifies dσ/σ as LCB does (κ·dσ): 2.5e-5 measured on an H100 at every scale
        scale = 1.0 if acq == "pi" else s
        assert dm <= 1e-6 * s and da <= (1e-5 if acq == "ei" else 5e-5) * scale, (c, s, dm, da)
    _close(engs)


@pytest.mark.parametrize("acq", ["ei", "lcb"])
def test_y_scale_unnormalized(acq):
    """normalize_y off: the GP models the raw targets (prior mean 0), so μ_n itself is at the scale of y."""
    X, y0, Xc = _data()
    engs = _engines(acq, normalize_y=False)
    for c, s in [(0.0, 1.0), (1e3, 1.0), (2e4, 5.0)]:
        _same_decision(engs, X, c + s * y0, Xc, f"{acq} raw c={c:g} s={s:g}")
    _close(engs)


# ---- (b) adversarial near-ties at the calibration rows ------------------------------------------------------------------
def _near_tie_grid(X, y, Xc, acq, spread=2e-3, n_ties=96):
    """Copies of the oracle's winner moved along a line through it, to the line's maximum and to points whose true acquisition
    values spread over `spread` below that maximum, placed at the stratified calibration rows ⌊i·M/n⌋ (n = 64 per SM, as the
    sweep samples them) and at other rows."""
    th = O.theta_of_record(D)
    fit = O.gp_fit(X, y, kind=KIND, length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    y_opt = float(np.min(y))
    mu, sd = O.gp_predict(fit, Xc)
    a = O.acquisition(mu, sd, y_opt, acq, th["xi"], th["kappa"])
    w = Xc[int(np.argmax(a))]
    rng = np.random.default_rng(11)
    u = rng.standard_normal(D)
    cand = np.clip(w + np.linspace(-0.05, 0.05, 20001)[:, None] * (u / np.linalg.norm(u)), 0.0, 1.0)
    mc, sc = O.gp_predict(fit, cand)
    ac = O.acquisition(mc, sc, y_opt, acq, th["xi"], th["kappa"])
    top = float(ac.max())
    assert top >= float(a.max())
    pick = np.flatnonzero(ac > top - spread)
    assert len(pick) >= n_ties, f"only {len(pick)} points of the line within {spread:g} of its maximum"
    pick = pick[np.argsort(ac[pick])][np.linspace(0, len(pick) - 1, n_ties).astype(int)]     # spread over the whole window
    ties = cand[pick]
    G = Xc.copy()
    n_cal = min(M, torch.cuda.get_device_properties(0).multi_processor_count * 64)
    cal = (np.arange(n_cal, dtype=np.int64) * M) // n_cal
    rows = np.concatenate([cal[np.linspace(0, n_cal - 1, n_ties // 2).astype(int)], rng.choice(M, n_ties - n_ties // 2, replace=False)])
    G[rows] = ties
    mg, sg = O.gp_predict(fit, G)
    ag = O.acquisition(mg, sg, y_opt, acq, th["xi"], th["kappa"])
    order = np.sort(ag)[::-1]
    assert order[0] - order[n_ties // 2] < spread and order[0] - order[n_ties // 2] > 0, "near-ties not in place"
    return G, ag


@pytest.mark.parametrize("acq", ["ei", "lcb"])
@pytest.mark.parametrize("c,s", [(2e4, 5.0), (-1e5, 2.0)])
def test_near_ties_at_the_calibration_rows(c, s, acq):
    X, y0, Xc = _data()
    y = c + s * y0
    G, ag = _near_tie_grid(X, y, Xc, acq, spread=2e-3 * s)
    engs = _engines(acq)
    b6 = _same_decision(engs, X, y, G, f"near-ties {acq} c={c:g} s={s:g}")
    i = int(np.argmax(ag))
    assert abs(b6.value - ag[i]) <= 1e-8 * max(1.0, abs(ag[i]))
    assert b6.index == i or ag[i] - ag[b6.index] <= 1e-8 * max(1.0, abs(ag[i]))
    _close(engs)


# ---- (c) the θ range --------------------------------------------------------------------------------------------------
THETAS = [("amp0.01", dict(amplitude=0.01)), ("amp1000", dict(amplitude=1000.0)), ("amp1e5", dict(amplitude=1e5)),
          ("noise0", dict(noise=0.0)), ("noise1e-6", dict(noise=1e-6)), ("noise0.1", dict(noise=0.1)),
          ("ls0.2", dict(ls_mult=0.2)), ("ls5", dict(ls_mult=5.0)), ("ls5-noise1e-6", dict(ls_mult=5.0, noise=1e-6))]
# Bounds on max |acq(tensor cores, three products) − acq(FP64)| over the grid (DESIGN.md §1): the 1e-5 contract (5e-5 for LCB,
# κ·dσ) where it holds, a small multiple of the value measured on an H100 where it does not.  The error of σ² grows with the
# amplitude (measured at 1000: 2.5e-4 EI, 1.3e-3 LCB); long length scales make σ small where dσ² is not, and κ·dσ grows as
# dσ²/σ (2.4e-4 LCB at ℓ×5; 4.2e-3 LCB and 1.6e-2 EI at ℓ×5 with noise 1e-6, at a winner with σ ≈ 5e-3).  Amplitude 1e5 takes
# the FP64 path in every mode, so the 'tc' engine's arrays there are the FP64 engine's.
ARRAY_TOL = {("amp1000", "ei"): 1e-3, ("amp1000", "lcb"): 5e-3, ("amp1e5", "ei"): 1e-10, ("amp1e5", "lcb"): 1e-10,
             ("ls5", "lcb"): 1e-3, ("ls5-noise1e-6", "lcb"): 1.5e-2, ("ls5-noise1e-6", "ei"): 5e-2}
# The suggestion's value against the FP64 engine's: 1e-10 relative, except where the two FP64 evaluations (panel solves with L
# against a product with W = L⁻¹) differ by more — at ℓ×5 with noise 1e-6 the FP64 oracle's own mean is off by 1e-9 against a
# long-double fit (test_fp64_engine_against_long_double).
VALUE_RTOL = {"ls5-noise1e-6": 1e-8}


def _theta(over):
    over = dict(over)
    m = over.pop("ls_mult", 1.0)
    return dict(over, length_scale=O.theta_of_record(D)["length_scale"] * m)


def _outcome(fn):
    from kubeflow_b200 import _lib as Lb
    try:
        return fn(), None
    except Lb.KboNotPositiveDefinite as e:
        return None, type(e)


@pytest.mark.parametrize("acq", ["ei", "lcb"])
@pytest.mark.parametrize("name,over", THETAS, ids=[t[0] for t in THETAS])
def test_theta_range(name, over, acq):
    X, y, Xc = _data()
    engs = _engines(acq, **_theta(over))
    outs = {}
    for k, e in engs.items():
        outs[k] = _outcome(lambda: e.tell(X, y).ask(Xc))
    errs = {k: o[1] for k, o in outs.items()}
    assert len(set(errs.values())) == 1, f"{name}: engines disagree on positive definiteness: {errs}"
    if errs["f64"] is not None:
        _close(engs)
        return
    b6 = outs["f64"][0]
    for k in VARIANTS:
        _check_same(k, engs[k], outs[k][0], b6, f"{name}/{acq}", VALUE_RTOL.get(name, 1e-10))
    # the per-candidate arrays of the three-product sweep against the FP64 engine's
    _, mu6, sd6, a6 = engs["f64"].ask(Xc, return_arrays=True)
    _, mut, sdt, at = engs["tc"].ask(Xc, return_arrays=True)
    da = float((at - a6).abs().max())
    print(f"\n{name}/{acq}: max|d acq| {da:.3e} max|d mu| {float((mut - mu6).abs().max()):.3e} max|d std| {float((sdt - sd6).abs().max()):.3e}")
    assert torch.isfinite(at).all()
    assert da <= ARRAY_TOL.get((name, acq), 5e-5 if acq == "lcb" else 1e-5)
    _close(engs)


# ---- (d) the FP64 engine against a long-double restatement ----------------------------------------------------------------
def _kernel_ld(A, B, ls, amp):
    A = np.asarray(A, dtype=np.longdouble) / np.asarray(ls, dtype=np.longdouble)
    B = np.asarray(B, dtype=np.longdouble) / np.asarray(ls, dtype=np.longdouble)
    d2 = ((A[:, None, :] - B[None, :, :]) ** 2).sum(-1)
    s = np.sqrt(np.longdouble(5) * d2)
    return np.longdouble(amp) * (1 + s + s * s / 3) * np.exp(-s)


def _predict_ld(X, y, Xc, ls, amp, noise):
    """fit + predict in long double: column-loop Cholesky, forward substitution, back substitution."""
    X = np.asarray(X, dtype=np.longdouble)
    y = np.asarray(y, dtype=np.longdouble)
    ym = y.mean()
    ys = np.sqrt(((y - ym) ** 2).mean())
    yn = (y - ym) / ys
    n = len(y)
    K = _kernel_ld(X, X, ls, amp) + np.longdouble(noise) * np.eye(n, dtype=np.longdouble)
    Lm = np.zeros_like(K)
    for j in range(n):
        d = K[j, j] - (Lm[j, :j] ** 2).sum()
        if not d > 0:
            return None
        Lm[j, j] = np.sqrt(d)
        Lm[j + 1:, j] = (K[j + 1:, j] - Lm[j + 1:, :j] @ Lm[j, :j]) / Lm[j, j]

    def fwd(B):   # L⁻¹ B
        Z = np.zeros_like(B)
        for i in range(n):
            Z[i] = (B[i] - Lm[i, :i] @ Z[:i]) / Lm[i, i]
        return Z

    z = fwd(yn[:, None])[:, 0]
    alpha = np.zeros(n, dtype=np.longdouble)
    for i in range(n - 1, -1, -1):
        alpha[i] = (z[i] - Lm[i + 1:, i] @ alpha[i + 1:]) / Lm[i, i]
    Ks = _kernel_ld(Xc, X, ls, amp)
    V = fwd(Ks.T.copy())
    var = np.maximum(np.longdouble(amp) - (V * V).sum(0), 0)
    return ym + ys * (Ks @ alpha), ys * np.sqrt(var), y.min()


LD_THETAS = [("noise0", dict(noise=0.0)), ("noise1e-6", dict(noise=1e-6)), ("ls5-noise1e-6", dict(ls_mult=5.0, noise=1e-6)),
             ("amp1e5-noise1e-6", dict(amplitude=1e5, noise=1e-6))]


@pytest.mark.skipif(np.finfo(np.longdouble).eps == np.finfo(np.float64).eps, reason="long double is double on this platform")
@pytest.mark.parametrize("acq", ["ei", "lcb"])
@pytest.mark.parametrize("name,over", LD_THETAS, ids=[t[0] for t in LD_THETAS])
def test_fp64_engine_against_long_double(name, over, acq):
    """Ill-conditioned θ at N = 256: the FP64 engine's μ, σ and acquisition within 4× the FP64 oracle's own error against a
    long-double fit and predict, plus 1e-12 of the values' magnitude (at amplitude 1e5, σ² = amplitude − Σv² cancels at the scale
    of 1e5: the summation order alone gives 5× the oracle's error of 1e-11 there).  The LCB reference is evaluated in long double;
    the EI reference is the float64 acquisition of the long-double μ and σ (SciPy's normal CDF has no long-double version)."""
    from kubeflow_b200.gp import GPEngine
    X, y, Xc = O.synthetic(256, 2000, 4)
    th = {**O.theta_of_record(4), **over}
    th["length_scale"] = O.theta_of_record(4)["length_scale"] * th.pop("ls_mult", 1.0)
    ref = _predict_ld(X, y, Xc, th["length_scale"], th["amplitude"], th["noise"])
    if ref is None:
        pytest.skip(f"{name}: the Gram matrix is not positive definite in long double either")
    mu_l, sd_l, yo = ref
    a_l = O.acquisition(mu_l.astype(np.float64), sd_l.astype(np.float64), float(yo), acq, th["xi"], th["kappa"])   # for the scale only
    try:
        orc = O.suggest(X, y, Xc, kind=KIND, acq=acq, **th)
    except np.linalg.LinAlgError:
        pytest.skip(f"{name}: the FP64 oracle's Cholesky fails")
    eng = GPEngine(0, kernel=KIND, acq=acq, var_mode="f64", **th)
    eng.tell(X, y)
    b, mu, sd, a = eng.ask(Xc, return_arrays=True)
    mu, sd, a = mu.cpu().numpy(), sd.cpu().numpy(), a.cpu().numpy()

    def acq_ld(m, s):   # the acquisition of long-double μ, σ, evaluated in long double where the formula allows
        m, s = np.asarray(m, dtype=np.longdouble), np.asarray(s, dtype=np.longdouble)
        if acq == "lcb":
            return -(m - np.longdouble(th["kappa"]) * s)
        return a_l
    ref_a = acq_ld(mu_l, sd_l)
    for what, got, want, oracle in (("mu", mu, mu_l, orc["mu"]), ("std", sd, sd_l, orc["std"]), ("acq", a, ref_a, orc["acq"])):
        e_gpu = float(np.abs(got - want).max())
        e_orc = float(np.abs(oracle - want).max())
        floor = 1e-12 * max(1.0, float(np.abs(want).max()))    # relative to the values' scale: σ ~ √amplitude
        print(f"\n{name}/{acq} {what}: |gpu − ld| {e_gpu:.3e}  |oracle − ld| {e_orc:.3e}")
        assert e_gpu <= 4 * e_orc + floor, (what, e_gpu, e_orc)
    eng.close()


# ---- (e) the standalone fp32 pass at a raw y scale ------------------------------------------------------------------------
@pytest.mark.parametrize("acq", ["ei", "lcb", "pi"])
def test_acq_argmax_f32_standalone_at_a_raw_y_scale(acq):
    """kbo_acq_argmax with y_mean = 2e4, y_std = 5: the values must carry the normalised posterior's accuracy, scaled by y_std,
    not fp32 rounding at the scale of y_mean."""
    from kubeflow_b200.gp import GPEngine
    r = np.random.default_rng(3)
    Mc = 1_000_003
    mu_n = r.standard_normal(Mc).astype(np.float32)
    var_n = (r.random(Mc) * 0.5).astype(np.float32)
    ym, ys = 2e4, 5.0
    yo = ym + ys * (-1.1 - 0.2) / 0.7
    mu = ym + ys * mu_n.astype(np.float64)
    sd = ys * np.sqrt(np.maximum(var_n.astype(np.float64), 0))
    ref = O.acquisition(mu, sd, yo, acq, 0.01, 1.96)
    eng = GPEngine(0, acq=acq)
    out = torch.empty(Mc, dtype=torch.float32, device="cuda")
    b = eng.acq_argmax_f32(torch.tensor(mu_n, device="cuda"), torch.tensor(var_n, device="cuda"), y_mean=ym, y_std=ys, y_opt=yo,
                           acq_out=out, global_offset=10)
    got = out.cpu().numpy().astype(np.float64)
    scale = 1.0 if acq == "pi" else ys
    if acq == "lcb":   # the fp32 output holds the raw value (≈ −y_mean): its own rounding is ulp(2e4) / 2
        np.testing.assert_allclose(got, ref, rtol=0, atol=2e-6 * scale + 1e-3)
    else:
        np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-6 * scale)
    i = int(np.argmax(ref))
    assert b.index - 10 == i or abs(ref[b.index - 10] - ref[i]) < 2e-6 * scale, (b.index - 10, i, ref[b.index - 10] - ref[i])
    assert abs(b.value - ref[i]) < 2e-6 * scale + 1e-5 * abs(ref[i]) * (acq != "lcb") + 1e-3 * (acq == "lcb")
    eng.close()


# ---- NaN: defined outcomes, and no pruning on a bound that lost its σ ---------------------------------------------------------
@pytest.mark.parametrize("acq", ["ei", "lcb"])
def test_nan_candidates_at_the_calibration_rows(acq):
    """NaN candidate rows at the stratified calibration rows make the calibrated E and Eμ NaN.  The bounds must then be NaN
    (nothing is pruned, the sweep falls back) — not σ-blind bounds at σ = 0, which for LCB prune on μ alone against a lower bound
    that includes κσ.  Every variant must return the FP64 engine's suggestion, which skips the NaN rows."""
    X, y0, Xc = _data()
    G = Xc.copy()
    n_cal = min(M, torch.cuda.get_device_properties(0).multi_processor_count * 64)
    cal = (np.arange(n_cal, dtype=np.int64) * M) // n_cal
    G[cal[::97]] = np.nan
    G[np.random.default_rng(5).choice(M, 64, replace=False)] = np.nan
    engs = _engines(acq)
    b6 = _same_decision(engs, X, 2e4 + 5 * y0, G, f"NaN rows {acq}")
    assert not np.isnan(G[b6.index]).any()
    _close(engs)


@pytest.mark.parametrize("acq", ["ei", "lcb"])
def test_nan_objective_gives_the_fp64_engines_outcome(acq):
    """A NaN objective makes y_mean, and with it every mean and acquisition value, NaN: nothing can be picked.  Every variant,
    array-free or returning arrays, must report what the FP64 engine reports — no pick (value −inf) — rather than read past the
    grid at the no-pick index."""
    X, y0, Xc = _data()
    y = y0.copy()
    y[7] = np.nan
    engs = _engines(acq)
    for e in engs.values():
        e.tell(X, y)
    b6 = engs["f64"].ask(Xc[:5000])
    assert b6.value == -np.inf
    for name in VARIANTS:
        b = engs[name].ask(Xc[:5000])
        assert (b.index, b.value) == (b6.index, b6.value), (name, b, b6)
    ba, _, _, a = engs["tc"].ask(Xc[:5000], return_arrays=True)
    assert (ba.index, ba.value) == (b6.index, b6.value) and torch.isnan(a).all()
    _close(engs)


def test_acq_argmax_rejects_a_non_positive_y_std():
    """The standalone pass ranks in units of y_std: 0, a negative or a non-finite y_std is an invalid argument."""
    from kubeflow_b200 import _lib as Lb
    from kubeflow_b200.gp import GPEngine
    eng = GPEngine(0, acq="ei")
    mu = torch.zeros(16, dtype=torch.float32, device="cuda")
    var = torch.ones(16, dtype=torch.float32, device="cuda")
    for ys in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(Lb.KboInvalidArgument):
            eng.acq_argmax_f32(mu, var, y_mean=0.0, y_std=ys, y_opt=-1.0)
    eng.close()
