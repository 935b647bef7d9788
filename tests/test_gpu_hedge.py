"""GPU: what gp_hedge runs on.  kbo_sweep_multi against one kbo_sweep per acquisition on the same fit and grid, in every sweep
variant of test_gpu_theta_range.py and the FP64 mode; kbo_predict_mean against the oracle; the Optimizer with the real engine
against the host replay of test_hedge_host.py; and the service with its default settings (acq_func = gp_hedge)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O
from tests.test_gpu_theta_range import D, KIND, M, N, VARIANTS, _data, _near_tie_grid

pytestmark = pytest.mark.gpu

ALL_VARIANTS = {**{k: dict(var_mode="tc", **v) for k, v in VARIANTS.items()}, "f64": dict(var_mode="f64")}


def _engine(over, normalize_y=True):
    from kubeflow_b200.gp import GPEngine
    return GPEngine(0, kernel=KIND, acq="ei", normalize_y=normalize_y, **O.theta_of_record(D), **over)


def _same(b, s, label):
    """One acquisition of the multi sweep against its single sweep: same index; value, μ, σ to 1e-12 relative."""
    assert b.index == s.index, f"{label}: index {b.index} vs {s.index}"
    for f in ("value", "mu", "std"):
        x, y = getattr(b, f), getattr(s, f)
        if np.isfinite(y):
            assert abs(x - y) <= 1e-12 * max(1.0, abs(y)), f"{label}: {f} {x!r} vs {y!r}"
        else:
            assert x == y, f"{label}: {f} {x!r} vs {y!r}"


def _compare(e, X, y, Xc, acqs, label, goff=0):
    """Fresh fit before every sweep, so each one starts from the same (lazy) state."""
    e.tell(X, y)
    multi = e.ask_multi(Xc, acqs, global_offset=goff)
    dec = e.last_decisions()
    assert len(dec) == len(acqs)
    for k, a in enumerate(acqs):
        e.acq = a
        e.tell(X, y)
        s = e.ask(Xc, global_offset=goff)
        lab = f"{label} {a} (of {acqs})"
        _same(multi[k], s, lab)
        single = (e.last_unrefined(), e.last_contenders(), e.last_prefix_survivors())
        assert e.last_decisions() == [single]
        # decided at the same stage: the same unrefined / contenders / prefix-survivor counts as the single sweep (the FP64
        # mode refines nothing, and kbo_last_contenders keeps whatever an earlier tensor-core sweep left there)
        want = single if e.var_mode != "f64" else (single[0], dec[k][1], single[2])
        assert dec[k] == want, f"{lab}: decision {dec[k]} vs single sweep {single}"
    e.acq = "ei"
    return multi, dec


def _cal_rows():
    n_cal = min(M, torch.cuda.get_device_properties(0).multi_processor_count * 64)
    return (np.arange(n_cal, dtype=np.int64) * M) // n_cal


@pytest.mark.parametrize("variant", list(ALL_VARIANTS))
def test_sweep_multi_equals_single_sweeps(variant):
    X, y0, Xc = _data()
    e = _engine(ALL_VARIANTS[variant])
    for c, s in [(0.0, 1.0), (2e4, 5.0), (-1e5, 2.0)]:
        _compare(e, X, c + s * y0, Xc, ["ei", "lcb", "pi"], f"{variant} y={c:g}+{s:g}y0")
    y = 2e4 + 5.0 * y0
    G, _ = _near_tie_grid(X, y, Xc, "ei", spread=1e-2)
    _compare(e, X, y, G, ["lcb", "ei"], f"{variant} near-ties")
    Gn = Xc.copy()
    Gn[_cal_rows()[::7]] = np.nan
    _compare(e, X, y0, Gn, ["pi", "ei", "lcb"], f"{variant} NaN rows")
    flat = 0.5 + 1e-4 * np.random.default_rng(3).random((M, D))      # a flat landscape: every fallback fires
    _, dec = _compare(e, X, y0, flat, ["ei", "pi"], f"{variant} flat")
    if variant in ("tc", "tc-eager"):
        # the fallbacks fire: far more candidates than the lazy-fit solve cap pass the prefix bound
        assert all(d[2] > 256 for d in dec), dec
    dev = torch.tensor(Xc, device="cuda")
    _compare(e, X, y0, dev.float(), ["lcb"], f"{variant} f32 device offset", goff=123457)
    _compare(e, X, y0, Xc.astype(np.float32), ["pi", "lcb"], f"{variant} f32 host")
    _compare(e, X, y0, dev, ["pi", "lcb", "ei"], f"{variant} f64 device")
    e.close()


def test_sweep_multi_rejects_bad_requests():
    from kubeflow_b200 import _lib as L
    X, y0, Xc = _data()
    e = _engine({})
    e.tell(X[:256], y0[:256])
    with pytest.raises(L.KboInvalidArgument):
        e.ask_multi(Xc[:1000], ["ei", "ei"])
    with pytest.raises(L.KboInvalidArgument):
        e.ask_multi(Xc[:1000], ["ei", "lcb", "pi", "lcb"])
    out = torch.empty(8, dtype=torch.float64, device="cuda")
    g = np.ascontiguousarray(Xc[:1000])
    for kinds in ([0, 7], [-1]):
        arr = (C.c_int32 * len(kinds))(*kinds)
        rc = e.lib.kbo_sweep_multi(e._h, g.ctypes.data, L.KBO_F64, 1000, 0, 1, len(kinds), arr, out.data_ptr(), e._stream())
        assert rc == L.KBO_ERR_INVALID
    e.close()


@pytest.mark.parametrize("variant", ["tc", "f64"])
def test_predict_mean_against_the_oracle(variant):
    X, y0, Xc = _data()
    y = 2e4 + 5.0 * y0
    th = O.theta_of_record(D)
    e = _engine(ALL_VARIANTS[variant])
    P = Xc[:37]

    def check(Xh, yh):
        fit = O.gp_fit(Xh, yh, kind=KIND, length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
        want = O.gp_predict(fit, P)[0]
        for pts in (P, P.astype(np.float32), torch.tensor(P, device="cuda")):
            got = e.predict_mean(pts)
            ref = want if not (isinstance(pts, np.ndarray) and pts.dtype == np.float32) else O.gp_predict(fit, P.astype(np.float32))[0]
            np.testing.assert_allclose(got, ref, rtol=1e-10, atol=0)

    e.tell(X[:2000], y[:2000])                   # lazy fit in the tensor-core mode
    check(X[:2000], y[:2000])
    for i in range(2000, 2005):
        e.append(X[i], y[i])
    check(X[:2005], y[:2005])
    y2 = y.copy()
    y2[:1990] += 3.0
    e.rebase(1990, y2[:1990])
    check(X[:1990], y2[:1990])
    e.close()


def test_gpu_optimizer_follows_the_host_replay():
    from kubeflow_b200.optimizer import Optimizer
    from tests.test_hedge_host import Replay, _dims, _f
    opt = Optimizer(_dims(), n_initial_points=3, acq_func="gp_hedge", random_state=7, n_points=2000, candidate_backend="numpy")
    rep = Replay(opt.space, 7, 3, 2000)
    told_X, told_y = [], []
    for step in range(8):
        k = 2 if step % 3 == 2 else 1
        got = opt.ask() if k == 1 else opt.ask(n_points=k)
        got = [got] if k == 1 else got
        Xt = opt.space.transform(told_X) if told_X else np.empty((0, 0))
        want = rep.ask(Xt, told_y, k)
        for g, w in zip(got, want):
            np.testing.assert_allclose(np.asarray(g, dtype=float), np.asarray(w, dtype=float), rtol=0, atol=0)
        np.testing.assert_allclose(opt.gains, rep.real.gains, rtol=1e-9, atol=1e-9)
        ys = [_f(p) for p in got]
        opt.tell(got, ys)
        told_X.extend(got)
        told_y.extend(ys)
    assert opt.gains.any()


def test_service_default_settings_run_gp_hedge():
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.service import SkoptService
    from tests.test_grpc_service import add_trial, make_experiment
    svc = SkoptService()
    exp = make_experiment("bayesianoptimization", {"n_initial_points": 1, "random_state": 4}, name="hedge-default")
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=3)
    n = 0
    gains = []
    for _ in range(3):
        rep = svc.get_suggestions(req)
        opt = svc._services["hedge-default"].skopt_optimizer
        assert opt.hedge and len(rep.parameter_assignments) == 3
        for pa in rep.parameter_assignments:
            v = {a.name: float(a.value) for a in pa.assignments}
            assert 0.01 <= v["x0"] <= 0.1 and -1 <= v["x1"] <= 1 and 10 <= v["x2"] <= 20 and 0 <= v["x3"] <= 5
            n += 1
            add_trial(req, f"t{n}", v, (v["x0"] - 0.05) ** 2 * 100 + v["x1"] ** 2 + ((v["x2"] - 15) / 5) ** 2)
        gains.append(opt.gains.copy())
    assert not gains[1].any() and gains[2].any()        # the first model-based round picks; the next one moves the gains
    exp2 = make_experiment("bayesianoptimization", {"n_initial_points": 1, "random_state": 5}, name="hedge-default")
    req.experiment.CopyFrom(exp2)                       # another fingerprint: a new optimizer, gains from zero
    svc.get_suggestions(req)
    opt2 = svc._services["hedge-default"].skopt_optimizer
    assert opt2 is not opt and not opt2.gains.any() and opt2.next_xs is not None
