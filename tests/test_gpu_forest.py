"""GPU: the RF / ET surrogates of ``bayesianoptimization`` (csrc/forest.cu) against scikit-learn's trees (tests/golden) and the
FP64 restatement oracle/forest_oracle.py.

Cases at the shapes of record take y on a grid of 2^-12 (tests/_forest_ref.dyadic_case): every sum the splitter forms is then
exact, so the device and the restatement break equal proxies the same way and trees must match bit for bit."""
import grpc
import numpy as np
import pytest
import torch
from scipy import stats

from kubeflow_b200.forest import ForestEngine
from oracle import forest_oracle as F
from tests._forest_ref import assert_same_tree, dyadic_case, golden_cases, golden_trees

pytestmark = pytest.mark.gpu


def _export_all(eng, draws=False):
    return [eng.export(t, with_draws=draws) for t in range(eng.n_trees)]


@pytest.mark.parametrize("path", golden_cases(), ids=lambda p: p.rsplit("/", 1)[-1])
def test_rf_trees_equal_sklearn_with_its_bootstrap_counts(path):
    z = np.load(path)
    ref = golden_trees(z)
    eng = ForestEngine(kind="RF", n_trees=len(ref), seed=0)
    eng.tell(z["X"], z["y"], counts=z["counts"])
    for t, tr in enumerate(ref):
        ex = eng.export(t)
        assert np.array_equal(ex["counts"], z["counts"][t])
        assert_same_tree(ex, tr, rtol=1e-12, where=f"tree {t}")
    mu, sd = eng.predict(z["Xc"])
    np.testing.assert_allclose(mu, z["mu"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(sd, z["sigma"], rtol=1e-12, atol=1e-12)
    eng.close()


def test_rf_at_the_shapes_of_record_equals_the_restatement_and_its_bootstrap():
    N, D, T, seed = 8192, 32, 100, 12345
    X, y = dyadic_case(np.random.default_rng(8), N, D)
    eng = ForestEngine(kind="RF", n_trees=T, seed=seed)
    eng.tell(X, y)
    counts = F.bootstrap_counts(N, T, seed)
    for t in range(T):
        assert np.array_equal(eng.export(t)["counts"], counts[t]), f"tree {t}: bootstrap counts"
    for t in (0, 41, 99):
        ex = eng.export(t)
        assert_same_tree(ex, F.build_tree(X, y, counts[t], kind="RF"), rtol=0, where=f"tree {t}")
        assert (ex["n_node_samples"][ex["left"] < 0] >= 3).all()
    tm = eng.last_timings()
    print(f"RF fit N={N} D={D} T={T}: {tm['fit_ms']:.1f} ms")
    eng.close()


def _node_minmax(tree, X):
    """min / max of every feature over each node's samples (ET: every sample is in the root)."""
    n, D = len(tree["left"]), X.shape[1]
    mn, mx = np.full((n, D), np.inf, np.float32), np.full((n, D), -np.inf, np.float32)
    members = {0: np.arange(len(X))}
    for k in range(n):
        r = members.pop(k)
        if tree["left"][k] < 0:
            continue
        mn[k], mx[k] = X[r].min(axis=0), X[r].max(axis=0)
        go = X[r, tree["feature"][k]].astype(np.float64) <= tree["threshold"][k]
        members[tree["left"][k]], members[tree["right"][k]] = r[go], r[~go]
    return mn, mx


def test_et_draws_equal_the_philox_restatement_and_trees_the_restatement():
    N, D, T, seed = 3000, 6, 8, 77
    X, y = dyadic_case(np.random.default_rng(4), N, D, grid=True)
    eng = ForestEngine(kind="ET", n_trees=T, seed=seed)
    eng.tell(X, y)
    ref = F.build_forest(X, y, kind="ET", n_trees=T, seed=seed)
    normalised = []
    for t in range(T):
        ex = eng.export(t, with_draws=True)
        assert (ex["counts"] == 1).all()
        assert_same_tree(ex, ref[t], rtol=0, where=f"ET tree {t}")
        mn, mx = _node_minmax(ex, X)
        inner = ex["left"] >= 0
        k = np.repeat(np.arange(len(inner)), D).reshape(-1, D)
        f = np.tile(np.arange(D), (len(inner), 1))
        const = mx <= (mn + F.FEATURE_THRESHOLD)
        want = np.where(inner[:, None] & ~const, F.et_threshold(F.et_uniform(seed, t, k, f), mn, mx), np.nan)
        assert np.array_equal(ex["draws"], want, equal_nan=True), f"tree {t}: drawn thresholds"
        # each split is its own draw for the chosen feature
        kk = np.flatnonzero(inner)
        assert np.array_equal(ex["threshold"][kk], ex["draws"][kk, ex["feature"][kk]])
        ok = inner[:, None] & ~const & (mx > mn)
        u = (ex["draws"][ok] - mn[ok].astype(np.float64)) / (mx[ok].astype(np.float64) - mn[ok].astype(np.float64))
        normalised.append(u[np.isfinite(u)])
    u = np.concatenate(normalised)
    assert len(u) > 2000
    assert stats.kstest(u, "uniform").pvalue > 1e-3
    eng.close()


def _candidates(rng, trees, M, D):
    """Uniform rows, with a share of them exactly on each split's fp32 neighbours (RD and RU of the FP64 threshold), integer-grid
    and one-hot values in columns 0 and 1."""
    Xc = rng.random((M, D)).astype(np.float32)
    Xc[: M // 8, 0] = rng.integers(0, 9, M // 8) / 8.0
    Xc[: M // 8, 1] = rng.integers(0, 2, M // 8)
    at = []
    for tr in trees:
        k = np.flatnonzero(tr["left"] >= 0)
        th = tr["threshold"][k]
        rd = th.astype(np.float32)
        rd = np.where(rd.astype(np.float64) > th, np.nextafter(rd, np.float32(-np.inf)), rd)
        ru = np.nextafter(rd, np.float32(np.inf))
        at += list(zip(tr["feature"][k], rd)) + list(zip(tr["feature"][k], ru))
    rows = rng.integers(M // 8, M, len(at))
    for r, (f, v) in zip(rows, at):
        Xc[r, f] = v
    return Xc


@pytest.mark.parametrize("kind,M", [("RF", 4096), ("ET", 4096), ("RF", 1 << 20)])
def test_predict_is_bit_identical_to_the_restatement_on_exported_trees(kind, M):
    N, D, T = 2000, 5, 20
    rng = np.random.default_rng(5)
    X, y = dyadic_case(rng, N, D, grid=True)
    y = y + rng.standard_normal(N) * 1e-3                      # non-dyadic: the sums of the sweep carry rounding
    eng = ForestEngine(kind=kind, n_trees=T, seed=3)
    eng.tell(X, y)
    trees = _export_all(eng)
    Xc = _candidates(rng, trees, M, D)
    (best,), mu_d, sd_d = eng.sweep(torch.from_numpy(Xc).cuda(), ["ei"], return_arrays=True)
    mu, sd = F.predict(trees, Xc)
    assert np.array_equal(mu_d.cpu().numpy(), mu)
    assert np.array_equal(sd_d.cpu().numpy(), sd)
    mu_p, sd_p = eng.predict(Xc[:1000])
    assert np.array_equal(mu_p, mu[:1000]) and np.array_equal(sd_p, sd[:1000])
    eng.close()


def _check_pick(b, acq, mu, sd, y_opt, xi=0.01, kappa=1.96):
    v = F.acquisition(acq, mu, sd, y_opt, xi, kappa)
    top = v.max()
    assert v[b.index] >= top - 1e-13 * max(abs(top), 1e-300), f"{acq}: picked {v[b.index]!r}, max {top!r}"
    same = np.flatnonzero((mu[: b.index] == mu[b.index]) & (sd[: b.index] == sd[b.index]))
    assert len(same) == 0, f"{acq}: index {b.index} has an earlier twin {same[:3]}"
    assert b.mu == mu[b.index] and b.std == sd[b.index]


@pytest.mark.parametrize("kind,M", [("RF", 65536), ("ET", 65536), ("RF", 1 << 20)])
def test_sweep_picks_the_first_maximum_for_each_acquisition_and_hedge(kind, M):
    N, D, T = 1500, 4, 30
    rng = np.random.default_rng(11)
    X, y = dyadic_case(rng, N, D, grid=True)
    eng = ForestEngine(kind=kind, n_trees=T, seed=1)
    eng.tell(X, y)
    trees = _export_all(eng)
    Xc = _candidates(rng, trees, M, D)
    Xd = torch.from_numpy(Xc).cuda()
    mu, sd = F.predict(trees, Xc)
    for acq in ("ei", "lcb", "pi"):
        (b,) = eng.sweep(Xd, [acq])
        _check_pick(b, acq, mu, sd, eng.y_opt)
    hedge = eng.sweep(Xd, ["ei", "lcb", "pi"], global_offset=1000)
    for acq, b in zip(("ei", "lcb", "pi"), hedge):
        assert b.index >= 1000
        b.index -= 1000
        _check_pick(b, acq, mu, sd, eng.y_opt)
        assert b.index == eng.sweep(Xd, [acq])[0].index
    eng.close()


def test_fit_and_sweep_are_bit_reproducible():
    X, y = dyadic_case(np.random.default_rng(2), 4000, 8)
    y = y + np.random.default_rng(3).standard_normal(4000) * 1e-3
    Xc = torch.rand(300000, 8, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    outs = []
    for _ in range(2):
        for kind in ("RF", "ET"):
            eng = ForestEngine(kind=kind, n_trees=50, seed=21)
            eng.tell(X, y)
            bests, mu, sd = eng.sweep(Xc, ["ei", "lcb", "pi"], return_arrays=True)
            outs.append((kind, [eng.export(t) for t in (0, 49)], [(b.value, b.index) for b in bests], mu.cpu().numpy(), sd.cpu().numpy()))
            eng.close()
    for a, b in zip(outs[:2], outs[2:]):
        for ta, tb in zip(a[1], b[1]):
            assert_same_tree(ta, tb, rtol=0)
        assert a[2] == b[2] and np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4])


def test_non_finite_y_is_invalid_and_tiny_histories_are_single_leaves():
    from kubeflow_b200 import _lib as L
    eng = ForestEngine(kind="RF", n_trees=10, seed=0)
    with pytest.raises(L.KboInvalidArgument):
        eng.tell(np.zeros((5, 2)), np.array([0.0, 1.0, np.nan, 2.0, 3.0]))
    for n in (1, 2, 5):
        eng.tell(np.random.default_rng(n).random((n, 2)), np.arange(n, dtype=np.float64))
        for t in range(10):
            assert len(eng.export(t)["left"]) == 1
    eng.tell(np.random.default_rng(0).random((40, 2)), np.full(40, 3.25))     # constant y: leaves only, sigma 0
    mu, sd = eng.predict(np.random.default_rng(1).random((10, 2)))
    assert (mu == 3.25).all() and (sd == 0).all()
    eng.close()


# ---- the service -------------------------------------------------------------------------------------------------------
def _mixed_experiment(est, acq, objective, name, n_initial=5, extra=None):
    from kubeflow_b200.suggestion import api_pb as api
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = objective
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "bayesianoptimization"
    settings = {"base_estimator": est, "n_initial_points": n_initial, "acq_func": acq, "random_state": 17, "n_points": 512,
                "candidate_backend": "numpy", **(extra or {})}
    for k, v in settings.items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, lst in (("lr", api.DOUBLE, "0.001", "0.1", None), ("layers", api.INT, "1", "8", None),
                                      ("opt", api.CATEGORICAL, None, None, ["sgd", "adam", "rmsprop"]), ("bn", api.CATEGORICAL, None, None, ["on", "off"])):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        if lst:
            p.feasible_space.list.extend(lst)
        else:
            p.feasible_space.min, p.feasible_space.max = lo, hi
    return e


def _loss(v):
    return (np.log10(float(v["lr"])) + 2.0) ** 2 + 0.1 * (int(v["layers"]) - 5) ** 2 + {"sgd": 0.5, "adam": 0.0, "rmsprop": 0.2}[v["opt"]] \
        + (0.1 if v["bn"] == "off" else 0.0)


@pytest.fixture()
def sweeps(monkeypatch):
    """Every sweep the service makes: the candidates, the acquisitions, the picks and the forest's trees at that moment."""
    rec = []
    orig = ForestEngine.sweep

    def spy(self, Xc, acqs, global_offset=0, return_arrays=False):
        out = orig(self, Xc, acqs, global_offset, return_arrays)
        rec.append(dict(Xc=np.asarray(Xc, np.float32).copy(), acqs=list(acqs), bests=out, y_opt=self.y_opt, N=self.N,
                        trees=_export_all(self), xi=self.xi, kappa=self.kappa))
        return out
    monkeypatch.setattr(ForestEngine, "sweep", spy)
    return rec


def _serve():
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService, SkoptService
    sk = SkoptService()
    server, port = serve(DispatchService([sk]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    return sk, server, ch, SuggestionStub(ch)


def _run(stub, exp, rounds, per_request=1, sign=1.0, loss=_loss):
    from kubeflow_b200.suggestion import api_pb as api
    from tests.test_grpc_service import add_trial
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=per_request)
    out = []
    for _ in range(rounds):
        reply = stub.GetSuggestions(req)
        for pa in reply.parameter_assignments:
            v = {a.name: a.value for a in pa.assignments}
            out.append(v)
            add_trial(req, f"t{len(out)}", v, sign * loss(v))
    return out


@pytest.mark.parametrize("est,acq,objective", [("RF", "EI", 1), ("ET", "LCB", 2), ("RF", "gp_hedge", 2), ("ET", "PI", 1)])
def test_service_suggestions_are_the_oracle_argmax(sweeps, est, acq, objective):
    from kubeflow_b200.suggestion import api_pb as api
    sk, server, ch, stub = _serve()
    name = f"forest-{est}-{acq}-{objective}"
    exp = _mixed_experiment(est, acq, objective, name)
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    pts = _run(stub, exp, 40, sign=1.0 if objective == api.MINIMIZE else -1.0)
    assert len(pts) == 40 and len(sweeps) == 35
    opt = sk._services[name].skopt_optimizer
    for s in sweeps:
        mu, sd = F.predict(s["trees"], s["Xc"])
        for a, b in zip(s["acqs"], s["bests"]):
            _check_pick(b, a, mu, sd, s["y_opt"], s["xi"], s["kappa"])
    # the suggestion is the picked candidate (gp_hedge: the one its draw chose)
    last = sweeps[-1]
    j = opt.last_hedge[2] if acq == "gp_hedge" else 0
    row = last["Xc"][last["bests"][j].index:last["bests"][j].index + 1].astype(np.float64)
    got = pts[-1]
    want = opt.space.inverse_transform(row)[0]
    assert abs(float(got["lr"]) - float(want[0])) <= 1e-12 * float(want[0]) and int(got["layers"]) == int(want[1])
    assert got["opt"] == want[2] and got["bn"] == want[3]
    ch.close()
    server.stop(0)


def test_service_constant_liar_replay_and_nan(sweeps):
    from kubeflow_b200.suggestion import api_pb as api
    sk, server, ch, stub = _serve()
    a = _run(stub, _mixed_experiment("RF", "EI", 1, "cl-a", n_initial=4), 6, per_request=3)
    b = _run(stub, _mixed_experiment("RF", "EI", 1, "cl-b", n_initial=4), 6, per_request=3)
    assert a == b                                                 # same random_state: the same suggestions
    # each point of a request refits: on the told history, then on it plus one and two lies y = min(y) (the first model-based
    # sweep is the second point of the second request: 3 told trials and one lie reach n_initial_points = 4)
    ns = [s["N"] for s in sweeps]
    assert ns == list(range(4, 18)) * 2
    for s in sweeps[:14]:                                         # a lie is min(y): the incumbent does not move
        assert s["y_opt"] == min(_loss(v) for v in a[: s["N"] - s["N"] % 3])
    # tiny histories (1 and 2 trials) are single leaves; constant y works
    c = _run(stub, _mixed_experiment("ET", "EI", 1, "tiny", n_initial=1), 3, loss=lambda v: 1.5)
    assert len(c) == 3 and all(len(t["left"]) == 1 for s in sweeps[-2:] for t in s["trees"])
    # a NaN objective is refused as bad input
    from tests.test_grpc_service import add_trial
    req = api.GetSuggestionsRequest(experiment=_mixed_experiment("ET", "EI", 1, "nan", n_initial=1), current_request_number=1)
    add_trial(req, "t0", {"lr": 0.01, "layers": 2, "opt": "adam", "bn": "on"}, float("nan"))
    with pytest.raises(grpc.RpcError) as ei:
        stub.GetSuggestions(req)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    ch.close()
    server.stop(0)
