"""GPU: ``kernel="hamming"`` — skopt's HammingKernel GP served by the engine's RBF kernel on the one-hot columns.

At D = 32 categorical dimensions with 1, 2, 3 and 7 categories (96 one-hot columns):
* ``lml_grad_batch`` through ``thetafit.engine_batch_fn(hamming=…)`` against ``oracle.hamming_oracle`` from N = 1 to 8192, and the
  skopt fit (three starts, lockstep) against the oracle's fit;
* the suggestion against the oracle's FP64 argmax over every candidate, at M = 65 536 and 2²⁰, for EI, LCB, PI and gp_hedge;
* the sweep-mode choice at the ends of the weights' bounds and just inside the tensor-core range;
* the Optimizer's own suggestion (its candidates, drawn with one-category dimensions among them) against the oracle, at the
  default weights, at weights of 1e5 on the one-category dimensions and after the skopt fit;
* append and rebase against a refit, and gRPC rounds.

The oracle's posterior over 2²⁰ candidates is restated in FP64 torch (``_posterior``: the same per-dimension mismatch sum,
K*·α and a triangular solve), checked against ``hamming_oracle.predict`` on the first rows.  A pick is accepted if it is the
oracle's first argmax, or a candidate whose oracle value lies within 1e-9 (relative) of the maximum: two correct FP64
evaluations of a near-tie may order it either way.
"""
import functools

import grpc
import numpy as np
import pytest
import torch

from kubeflow_b200 import hamming as HM
from kubeflow_b200 import thetafit as TF
from kubeflow_b200.gp import GPEngine
from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, SkoptService
from oracle import hamming_oracle as H
from tests.test_hamming_oracle import categorical_experiment, space_of

pytestmark = pytest.mark.gpu

CATS = [1, 2, 3, 7] * 8                       # D = 32, 96 one-hot columns
SP = space_of(CATS)
HMAP = HM.HammingMap(SP)
ACTIVE = int((np.array(CATS) >= 2).sum())    # dimensions that can differ


def _codes(r, n):
    return np.stack([r.integers(0, c, n) for c in CATS], axis=1).astype(np.float64)


def _one_hot(C, dtype=np.float64):
    return SP.transform(C.tolist()).astype(dtype)


@functools.lru_cache(maxsize=None)
def _history(N, seed=0):
    r = np.random.default_rng(seed)
    X = _codes(r, N)
    w = r.standard_normal(len(CATS)) * (r.random(len(CATS)) < 0.5)
    eff = [r.standard_normal(c) for c in CATS]
    y = sum(w[j] * eff[j][X[:, j].astype(int)] for j in range(len(CATS))) + 0.1 * r.standard_normal(N)
    return X, np.asarray(y, dtype=np.float64)


@functools.lru_cache(maxsize=None)
def _grid(M, seed=1):
    return _codes(np.random.default_rng(seed), M)


def _posterior(f, Xc, batch=65536):
    """hamming_oracle.predict in FP64 torch on the device (for 2²⁰ candidates)."""
    dev = "cuda"
    X = torch.as_tensor(f["X"], device=dev)
    l = torch.as_tensor(f["l"], device=dev)
    Lc = torch.as_tensor(f["L"], device=dev)
    al = torch.as_tensor(f["alpha"], device=dev)
    mu, sd = [], []
    for s in range(0, len(Xc), batch):
        C = torch.as_tensor(Xc[s:s + batch], device=dev)
        S = torch.zeros((len(C), len(X)), dtype=torch.float64, device=dev)
        for j in range(X.shape[1]):
            S += l[j] * (C[:, j, None] != X[None, :, j])
        Ks = f["amp"] * torch.exp(-S)
        V = torch.linalg.solve_triangular(Lc, Ks.T, upper=False)
        mu.append(f["y_mean"] + f["y_std"] * (Ks @ al))
        sd.append(f["y_std"] * torch.sqrt(torch.clamp(f["amp"] - (V * V).sum(0), min=0.0)))
    return torch.cat(mu).cpu().numpy(), torch.cat(sd).cpu().numpy()


def _theta(l, amp=1.0, noise=1e-3):
    return np.log(np.r_[amp, HMAP.weights(l), noise])


@functools.lru_cache(maxsize=None)
def _reference(N, M, key):
    l, amp, noise = _WEIGHTS[key]
    X, y = _history(N)
    f = H.fit(X, y, _theta(l, amp, noise))
    Xc = _grid(M)
    mu, sd = _posterior(f, Xc)
    m0, s0 = H.predict(f, Xc[:2048])
    # two FP64 evaluations agree to about κ(K)·eps: 1e-12 at moderate θ, ~1e-10 at l_j = 1e-5 (every kernel value ≈ 1, κ ≈ 2e6)
    K = f["amp"] * f["Kh"] + (f["noise"] + H.ALPHA) * np.eye(N)
    rel = max(1e-12, 4 * np.linalg.cond(K) * np.finfo(np.float64).eps)
    assert np.abs(mu[:2048] - m0).max() <= rel * max(1.0, np.abs(m0).max())
    assert np.abs(sd[:2048] - s0).max() <= rel * max(1.0, np.abs(s0).max())
    return f, mu, sd


r_ = np.random.default_rng(5)
_WEIGHTS = {"moderate": (r_.uniform(0.05, 0.5, len(CATS)), 1.0, 1e-3),
            "lower-bound": (1e-5, 1.0, 1e-3), "upper-bound": (1e5, 1.0, 1e-3),
            "inside-lo": (HM.TC_RANGE[0] * 1.02 / ACTIVE, 1.0, 1e-3), "inside-hi": (HM.TC_RANGE[1] * 0.98 / ACTIVE, 1.0, 1e-3)}


def _engine(key, acq="ei"):
    l, amp, noise = _WEIGHTS[key]
    e = GPEngine(0, kernel="rbf", acq=acq, length_scale=HMAP.length_scale(l), amplitude=amp, noise=noise + H.ALPHA,
                 var_mode=HMAP.var_mode(l, "auto"))
    return e.record_stages()


def _check_pick(b, acq, f, mu, sd, label):
    a = H.acquisition(mu, sd, float(np.min(f["y"])), acq, 0.01, 1.96)
    i = int(np.argmax(a))
    msg = f"{label}/{acq}: pick {b.index} ({a[b.index]!r}), oracle {i} ({a[i]!r})"
    assert b.index == i or a[b.index] >= a[i] - 1e-9 * max(1.0, abs(a[i])), msg
    j = b.index
    assert abs(b.mu - mu[j]) <= 1e-8 * max(1.0, abs(mu[j])) and abs(b.std - sd[j]) <= 1e-8 * max(1.0, sd[j]), (msg, b, mu[j], sd[j])


# ---- LML, gradient and the fit ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 64, 1000, 8192])
def test_lml_and_gradient_against_the_oracle(N):
    X, y = _history(N)
    e = GPEngine(0, kernel="rbf", scratch_limit=16 << 30)
    r = np.random.default_rng(N)
    thetas = [_theta(r.uniform(0.02, 2.0, len(CATS)), r.uniform(0.5, 3.0), 10 ** r.uniform(-3, -1)) for _ in range(2 if N < 8192 else 1)]
    got = TF.engine_batch_fn(e, _one_hot(X), y, hamming=HMAP)(thetas)
    for t, (f, g) in zip(thetas, got):
        fo, go = H.objective(X, y, t)
        assert abs(f - fo) <= 1e-9 * max(1.0, abs(fo)), (N, f, fo)
        assert np.abs(g - go).max() <= 1e-8 * max(1.0, np.abs(go).max()), (N, np.abs(g - go).max())
        assert (g[1:-1][np.array(CATS) == 1] == 0).all()          # one-category dimensions: zero gradient
    e.close()


@pytest.mark.parametrize("N", [1, 64, 512, 8192])
def test_skopt_fit_against_the_oracle(N):
    """The device fit reaches the oracle's optimum.  N ≤ 512: the oracle's own fit (SciPy's L-BFGS-B from the same starts on the
    oracle's objective); the LML to 1e-7 relative, and the fitted θ to 1e-3 on every coordinate where the LML is curved (the
    oracle's ∂²/∂θ_k² ≥ 1 by central differences, away from the bounds; the NumPy stand-in of the device agrees to 1e-6 there).
    Along the other coordinates — irrelevant dimensions, weights at a bound — the LML is flat and where L-BFGS-B stops depends
    on the last bits of each gradient.  N = 8192, where one oracle evaluation takes most of a minute and the oracle's fit hours:
    the oracle's LML at the device's θ is the device's, and above the winning start's."""
    X, y = _history(N)
    e = GPEngine(0, kernel="rbf", scratch_limit=16 << 30)
    seed = TF.estimator_seed(7)
    res = TF.fit(TF.engine_batch_fn(e, _one_hot(X), y, hamming=HMAP), len(CATS), seed, 2, ls_bounds=HM.LS_BOUNDS)
    fo, _ = H.objective(X, y, res.theta)
    assert abs(-fo - res.lml) <= 1e-9 * max(1.0, abs(res.lml))
    np.testing.assert_array_equal(res.theta[1:-1][np.array(CATS) == 1], res.starts[res.winner].theta0[1:-1][np.array(CATS) == 1])
    if N <= 512:
        ref = H.skopt_fit(X, y, seed=seed)
        assert abs(res.lml - ref["lml"]) <= 1e-7 * max(1.0, abs(ref["lml"])), (N, res.lml, ref["lml"])
        assert res.winner == ref["winner"]
        t, b, h = ref["theta"], H.log_bounds(len(CATS)), 1e-4
        compared = 0
        for k in range(len(t)):
            if not (t[k] - b[k, 0] > 1e-3 and b[k, 1] - t[k] > 1e-3):
                continue
            tp, tm = t.copy(), t.copy()
            tp[k] += h
            tm[k] -= h
            if (H.objective(X, y, tp)[1][k] - H.objective(X, y, tm)[1][k]) / (2 * h) >= 1.0:
                assert abs(res.theta[k] - t[k]) <= 1e-3, (N, k, res.theta[k], t[k])
                compared += 1
        assert compared >= (0 if N == 1 else 2), compared
    else:
        assert res.lml >= -H.objective(X, y, res.starts[res.winner].theta0)[0]
    e.close()


# ---- the suggestion over the whole candidate set -----------------------------------------------------------------------------
@pytest.mark.parametrize("N,M", [(2048, 65536), (1536, 1 << 20)])
def test_pick_against_the_fp64_argmax(N, M):
    X, y = _history(N)
    f, mu, sd = _reference(N, M, "moderate")
    Xc = torch.as_tensor(_one_hot(_grid(M), np.float32), device="cuda")
    for acq in ("ei", "lcb", "pi"):
        e = _engine("moderate", acq)
        e.tell(_one_hot(X), y)
        b = e.ask(Xc)
        assert e.stages(), "the moderate θ must take the tensor-core path"
        _check_pick(b, acq, f, mu, sd, f"N={N} M={M}")
        e.close()
    e = _engine("moderate")
    e.tell(_one_hot(X), y)
    for acq, b in zip(("ei", "lcb", "pi"), e.ask_multi(Xc, ["ei", "lcb", "pi"])):     # gp_hedge's one sweep
        _check_pick(b, acq, f, mu, sd, f"hedge N={N} M={M}")
    e.close()


@pytest.mark.parametrize("key,mode", [("lower-bound", "f64"), ("upper-bound", "f64"), ("inside-lo", "auto"), ("inside-hi", "auto")])
def test_sweep_mode_at_the_ends_of_the_range(key, mode):
    """At the weights' bounds (1e-5 and 1e5 everywhere) auto takes the FP64 path; just inside the tensor-core range it takes the
    tensor cores, and both return the oracle's pick."""
    N, M = 2048, 65536
    X, y = _history(N)
    f, mu, sd = _reference(N, M, key)
    assert HMAP.var_mode(_WEIGHTS[key][0], "auto") == mode
    Xc = torch.as_tensor(_one_hot(_grid(M), np.float32), device="cuda")
    for acq in ("ei", "lcb"):
        e = _engine(key, acq)
        e.tell(_one_hot(X), y)
        b = e.ask(Xc)
        assert bool(e.stages()) == (mode == "auto"), (key, acq)
        _check_pick(b, acq, f, mu, sd, key)
        e.close()


# ---- append / rebase, and the Optimizer -------------------------------------------------------------------------------------
@pytest.mark.parametrize("theta_fit", [None, "skopt"])
def test_append_and_rebase_pick_as_a_refit(theta_fit):
    X, y = _history(1100, seed=3)
    pts = [[SP.dimensions[j].categories[int(v)] for j, v in enumerate(row)] for row in X]
    kw = dict(kernel="hamming", n_initial_points=1, random_state=4, acq_func="gp_hedge", n_points=65536, theta_fit=theta_fit)
    inc, ref = Optimizer(SP, **kw), Optimizer(SP, incremental=False, **kw)
    seen, rebases = set(), []
    for lo, hi in ((0, 1090), (1090, 1092), (1092, 1100)):
        for o in (inc, ref):
            o.tell(pts[lo:hi], y[lo:hi].tolist())
        if inc._engine is not None and not rebases:    # count the engine's rebases (lies dropped / replaced by real trials)
            rebase = inc._engine.rebase
            rebases.append(0)

            def counted(*a, **k):
                rebases[0] += 1
                return rebase(*a, **k)
            inc._engine.rebase = counted
        a, b = inc.ask(n_points=3), ref.ask(n_points=3)
        assert a == b, (lo, hi, a, b)
        seen.add(inc.last_fit)
    assert {"append"} <= seen
    # at fixed θ the next request's real trials replace the lies in place; the skopt fit refits θ on a changed history instead
    assert (rebases[0] >= 2) if theta_fit is None else (rebases[0] == 0), rebases
    if theta_fit == "skopt":
        assert inc.last_theta["length_scale"].shape == (len(CATS),)
    for o in (inc, ref):
        o._engine.close()


@pytest.mark.parametrize("mode", ["default", "large-one-category-weights", "skopt"])
def test_optimizer_pick_with_one_category_dimensions(mode):
    """Optimizer.ask on the D = 32 space (8 one-category dimensions) over its own 65 536 sampled candidates: the pick and its
    (μ, σ) are the oracle's on those candidates' category codes, at the fitted or given weights."""
    X, y = _history(2048, seed=4)
    pts = [[SP.dimensions[j].categories[int(v)] for j, v in enumerate(row)] for row in X]
    kw = dict(kernel="hamming", n_initial_points=1, random_state=8, acq_func="EI", n_points=65536)
    l = 1.0
    if mode == "large-one-category-weights":
        l = kw["length_scale"] = np.where(np.array(CATS) == 1, 1e5, 0.3)
    if mode == "skopt":
        kw["theta_fit"] = "skopt"
    o = Optimizer(SP, **kw)
    o.tell(pts, y.tolist())
    seen, sweep = [], o._sweep
    o._sweep = lambda eng, cand, lo=0: (seen.append(cand.double().cpu().numpy()), sweep(eng, cand, lo))[1]
    x = o.ask()
    codes = np.asarray([[SP.dimensions[j].categories.index(v) for j, v in enumerate(p)] for p in SP.inverse_transform(seen[0])],
                       dtype=np.float64)
    np.testing.assert_array_equal(_one_hot(codes), seen[0])           # the candidates are encoded as the told rows
    if mode == "skopt":
        th = o.last_theta
        theta = np.log(np.r_[th["amplitude"], th["length_scale"], th["noise"]])
    else:
        theta = _theta(l, 1.0, 1e-3 - H.ALPHA)                         # the engine's diagonal is noise = 1e-3 exactly
    f = H.fit(X, y, theta)
    mu, sd = _posterior(f, codes)
    _check_pick(o.last_best, "ei", f, mu, sd, mode)
    assert x == [SP.dimensions[j].categories[int(v)] for j, v in enumerate(codes[o.last_best.index])]
    o._engine.close()


# ---- gRPC --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([SkoptService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _request(exp, trials, k):
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=k)
    for i, (vals, loss) in enumerate(trials):
        t = req.trials.add()
        t.name = f"t{i}"
        t.spec.objective.objective_metric_name = "loss"
        for n, v in vals.items():
            a = t.spec.parameter_assignments.assignments.add()
            a.name, a.value = n, str(v)
        t.status.condition = api.SUCCEEDED
        m = t.status.observation.metrics.add()
        m.name, m.value = "loss", str(loss)
    return req


FEASIBLE = {"optimizer": {"sgd", "adam", "rmsprop"}, "batch": {"16", "32", "64"}, "bn": {"on", "off"}}


@pytest.mark.parametrize("settings", [{"kernel": "hamming"}, {"kernel": "hamming", "theta_fit": "skopt"},
                                      {"kernel": "hamming", "acq_func": "LCB", "length_scale": 0.3}])
def test_grpc_rounds(stub, settings):
    s = {"n_initial_points": 1, "random_state": 11, **settings}
    trials = [({"optimizer": "adam", "batch": "32", "bn": "on"}, 0.4), ({"optimizer": "sgd", "batch": "16", "bn": "off"}, 0.9)]
    for n_hist in (1, 2):
        name = f"ham-{abs(hash(tuple(sorted(s.items()))))}-{n_hist}"
        exp = categorical_experiment(s, name=name)
        r1 = stub.GetSuggestions(_request(exp, trials[:n_hist], 3))      # constant liar for points 2 and 3
        assert len(r1.parameter_assignments) == 3
        for pa in r1.parameter_assignments:
            assert {a.name: a.value for a in pa.assignments}.keys() == FEASIBLE.keys()
            for a in pa.assignments:
                assert a.value in FEASIBLE[a.name]
        # replay: the same history to a new experiment of the same settings gives the same suggestions
        r2 = stub.GetSuggestions(_request(categorical_experiment(s, name=name + "-replay"), trials[:n_hist], 3))
        assert [[(a.name, a.value) for a in pa.assignments] for pa in r1.parameter_assignments] == \
               [[(a.name, a.value) for a in pa.assignments] for pa in r2.parameter_assignments]
