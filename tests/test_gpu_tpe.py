"""GPU: the TPE engine (kbo_tpe_*, kubeflow_b200.tpe.Tpe) against its FP64 contract, oracle/tpe_oracle.py — the models it builds,
the decision over caller-supplied candidates, its sampler, and the ``tpe`` service over gRPC."""
import grpc
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import tpe_oracle as O
from tests import _tpe_ref as R

pytestmark = pytest.mark.gpu

KINDS = [("uniform", -1.0, 3.0), ("quniform", 0.0, 20.0, 1.0), ("quniform", 3.0, 48.0, 5.0), ("choice", 3), ("choice", 64), ("choice", 4)]


def space_of(D):
    return [KINDS[0]] if D == 1 else [KINDS[d % len(KINDS)] for d in range(D)]


def history(space, n, seed):
    """n trials with tied values (a third of every uniform column on a 0.25 grid) and tied, non-finite losses."""
    r = np.random.default_rng(seed)
    X = np.empty((n, len(space)))
    for d, p in enumerate(space):
        if p[0] == "uniform":
            v = r.uniform(p[1], p[2], n)
            v[: n // 3] = np.round(v[: n // 3] * 4) / 4
        elif p[0] == "quniform":
            v = np.round(r.uniform(p[1], p[2], n) / p[3]) * p[3]
        else:
            v = r.integers(0, p[1], n).astype(float)
        X[:, d] = v
    losses = r.integers(0, max(n // 4, 2), n).astype(float)
    if n > 3:
        losses[1], losses[2] = np.nan, np.inf
    return X, losses


def engine(space, X, losses, seed=11, **kw):
    from kubeflow_b200.tpe import Tpe
    t = Tpe(space, seed=seed, **kw)
    t.tell(X, losses)
    return t


def _multiset(*cols):
    A = np.stack(cols, axis=1)
    return A[np.lexsort(A.T[::-1])]


@pytest.mark.parametrize("D", [1, 4, 32])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 25, 26, 27, 200, 8192])
def test_models_match_oracle(n, D):
    space = space_of(D)
    X, losses = history(space, n, seed=n * 100 + D)
    t = engine(space, X, losses)
    got = t.state()
    ref, nb = O.build_models(space, X, losses)
    for d, (g, m) in enumerate(zip(got, ref)):
        assert g["n_below"] == nb
        for grp in ("below", "above"):
            if m["kind"] == "choice":
                np.testing.assert_allclose(g[grp]["p"], m[grp], rtol=1e-13, atol=0)
                continue
            a, b = g[grp], m[grp]
            assert len(a["w"]) == len(b["w"]), (d, grp)
            np.testing.assert_allclose(_multiset(a["mu"], a["sigma"], a["w"]), _multiset(b["mu"], b["sigma"], b["w"]), rtol=1e-13, atol=0,
                                       err_msg=f"param {d} {grp}")
            assert abs(a["p_accept"] - b["p_accept"]) <= 1e-13 * b["p_accept"]
    t.close()


def _oracle_scores(model, x, chunk=2048):
    return np.concatenate([O.score(model, x[i:i + chunk]) for i in range(0, len(x), chunk)]) if len(x) else np.zeros(0)


def _first_best_level(model, c):
    """np.argmax over the candidates of a quantized / categorical parameter, evaluated once per distinct value: the first
    occurrence of the best-scoring value.  Returns (index, value)."""
    key = c if model["kind"] == "choice" else O.quantize(c, model["q"])
    u, first = np.unique(key, return_index=True)
    s = O.score(model, u)
    best = np.nan if np.isnan(s).any() else s.max()
    hit = np.isnan(s) if np.isnan(best) else s == best
    i = int(first[hit].min())
    return i, float(key[i])


SCORING_SPACE = [("uniform", -1.0, 3.0), ("quniform", 0.0, 20.0, 1.0), ("quniform", 3.0, 48.0, 5.0), ("choice", 64)]


@pytest.mark.parametrize("M", [24, 4096, 1 << 20])
@pytest.mark.parametrize("n", [20, 1000, 8192])
def test_decision_on_supplied_candidates(n, M):
    """Each parameter's winner is the oracle's np.argmax over the same candidates; every FP32 score lies within its bound of the
    FP64 score.  Up to M = 4096 the NumPy oracle scores every candidate; at M = 2^20 the continuous parameter's candidates are
    all scored by the FP64 torch restatement on the device (tests/_tpe_ref.py, pinned to the oracle by tests/test_tpe_ref.py),
    whose pick rule tells near-ties closer than two FP64 evaluations can separate from a wrong pick; the quantized and
    categorical parameters are scored exhaustively by the oracle, once per distinct value."""
    space = SCORING_SPACE
    X, losses = history(space, n, seed=n + 7)
    models, _ = O.build_models(space, X, losses)
    r = np.random.default_rng(M + n)
    cands = np.stack([O.draw(m, M, r) for m in models])
    if M >= 4096:
        cands[:, M // 2:] = cands[:, : M - M // 2]                    # every candidate twice: the first copy must win
    t = engine(space, X, losses)
    out = t.ask(1, M, candidates=torch.tensor(cands[None], device="cuda"), return_details=True)
    sc = out["scores"][0, 0].cpu().numpy().astype(np.float64)
    assert np.array_equal(out["candidates"][0].cpu().numpy(), cands)
    s32, e32 = sc[:, 0], sc[:, 1]
    if M <= 4096:
        s64 = _oracle_scores(models[0], cands[0])
        win0 = int(np.argmax(s64))
    else:
        x0 = out["candidates"][0, 0]
        s64_dev = R.score(models[0], x0)
        win0 = int(out["index"][0, 0])
        ok, msg, _ = R.pick_ok(models[0], x0, s64_dev, win0)
        assert ok, msg
        s64 = s64_dev.cpu().numpy()
    err = np.abs(s32 - s64)
    assert (err <= e32).all(), f"max excess {np.max(err - e32):.3e}"
    ref = [_first_best_level(m, c) for m, c in zip(models[1:], cands[1:])]
    if M <= 4096:
        assert O.choose(models[1:], cands[1:])[1].tolist() == [i for i, _ in ref]       # the literal np.argmax over candidates
    assert out["index"][0].tolist() == [win0] + [i for i, _ in ref]
    assert out["x"][0].tolist() == [cands[0, win0]] + [v for _, v in ref]
    if M >= 4096:
        assert (out["index"][0] < M // 2).all()
    print(f"\nn={n} M={M}: survivors (FP64 candidates / distinct values scored) {out['survivors'][0].tolist()}, "
          f"median bound {np.median(e32):.2e}, max |s32 - s64| {err.max():.2e}")
    t.close()


def test_all_tied_scores_pick_the_first_candidate():
    """No history: both models are the prior, every candidate of every parameter scores the same (exactly 0 in FP64), so the
    first candidate wins everywhere — the continuous parameter after an FP64 pass over all of them."""
    space = SCORING_SPACE
    t = engine(space, np.zeros((0, 4)), np.zeros(0))
    out = t.ask(2, 4096, return_details=True)
    assert (out["index"] == 0).all()
    assert out["survivors"][:, 0].tolist() == [4096, 4096]
    t.close()


def test_sampler_distribution_bounds_and_determinism():
    space = [("uniform", -1.0, 3.0), ("quniform", 3.0, 48.0, 5.0), ("choice", 4)]
    X, losses = history(space, 300, seed=5)
    t = engine(space, X, losses, seed=2024)
    M = 1 << 20
    out = t.ask(1, M, return_details=True)
    C = out["candidates"][0].cpu().numpy()
    st = t.state()
    for d, (lo, hi) in ((0, (-1.0, 3.0)), (1, (3.0, 48.0))):
        assert (C[d] >= lo).all() and (C[d] < hi).all()
        b = st[d]["below"]
        ks = stats.kstest(C[d], lambda x: O.truncated_mixture_cdf(x, b["w"], b["mu"], b["sigma"], lo, hi))
        assert ks.statistic < 1.95 / np.sqrt(M), ks                 # the 1e-3-level critical value; fixed seed, deterministic
    assert out["x"][0, 1] % 5.0 == 0.0
    counts = np.bincount(C[2].astype(int), minlength=4) / M
    assert np.abs(counts - st[2]["below"]["p"]).max() < 5e-3
    t2 = engine(space, X, losses, seed=2024)
    again = t2.ask(1, M, return_details=True)                     # same key (seed, ask 0): bit-identical
    assert np.array_equal(again["candidates"][0].cpu().numpy(), C) and np.array_equal(again["x"], out["x"])
    nxt = t2.ask(1, M, return_details=True)["candidates"][0].cpu().numpy()   # next ask counter: new draws
    assert not np.array_equal(nxt[0], C[0])
    t.close()
    t2.close()


# ---- the service over gRPC --------------------------------------------------------------------------------------------------
def _experiment(name, settings, dmax="3.0"):
    from kubeflow_b200.suggestion import api_pb as api
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MAXIMIZE
    e.spec.objective.objective_metric_name = "acc"
    e.spec.algorithm.algorithm_name = "tpe"
    for k, v in settings.items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, step, lst in (("x", api.DOUBLE, "-1.0", dmax, "", ()), ("layers", api.INT, "3", "48", "5", ()),
                                            ("opt", api.CATEGORICAL, None, None, "", ("sgd", "adam", "ftrl")),
                                            ("bs", api.DISCRETE, None, None, "", ("16", "32", "64"))):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        if lo is not None:
            p.feasible_space.min, p.feasible_space.max = lo, hi
        if step:
            p.feasible_space.step = step
        p.feasible_space.list.extend(lst)
    return e


def _objective(a):
    return -(float(a["x"]) - 1.3) ** 2 - 0.01 * abs(int(a["layers"]) - 23) + {"sgd": 0.0, "adam": 0.3, "ftrl": 0.1}[a["opt"]] \
        + 0.001 * int(a["bs"])


def _units(a):
    return [float(a["x"]), float(a["layers"]), float(["sgd", "adam", "ftrl"].index(a["opt"])), float(["16", "32", "64"].index(a["bs"]))]


@pytest.fixture(scope="module")
def tpe_stub():
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    from kubeflow_b200.suggestion.tpe_service import TpeService
    svc = TpeService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


def _run(stub, name, rounds, settings, check=None):
    from kubeflow_b200.suggestion import api_pb as api
    exp = _experiment(name, settings)
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=1)
    replies = []
    for i in range(rounds):
        rep = stub.GetSuggestions(req)
        a = {x.name: x.value for x in rep.parameter_assignments[0].assignments}
        replies.append(a)
        if check:
            check(i, a)
        t = req.trials.add()
        t.name = f"{name}-t{i}"
        t.spec.objective.objective_metric_name = "acc"
        for k, v in a.items():
            x = t.spec.parameter_assignments.assignments.add()
            x.name, x.value = k, v
        t.status.condition = api.SUCCEEDED
        m = t.status.observation.metrics.add()
        m.name, m.value = "acc", repr(_objective(a))
    return replies, req


def test_service_rounds_match_oracle_and_replay(tpe_stub):
    """20 start-up rounds and 60 model-based rounds on a mixed 4-D space.  A replica engine with the same seed, history and ask
    count regenerates the service's candidates; every model-based reply equals the oracle's choice over them."""
    from kubeflow_b200.suggestion.tpe_service import tpe_space
    from kubeflow_b200.suggestion.internal import HyperParameterSearchSpace
    from kubeflow_b200.tpe import Tpe
    stub, svc = tpe_stub
    settings = {"random_state": 42, "n_EI_candidates": 64}
    space = tpe_space(HyperParameterSearchSpace.convert(_experiment("svc-a", settings)))
    rows, losses = [], []
    replica = Tpe(space, seed=42)
    told = [0]

    def check(i, a):
        if i >= 20:
            if told[0] < len(rows):
                replica.tell(np.asarray(rows[told[0]:]), np.asarray(losses[told[0]:]))
                told[0] = len(rows)
            out = replica.ask(1, 64, return_details=True)
            models, _ = O.build_models(space, np.asarray(rows), np.asarray(losses))
            vals, _ = O.choose(models, out["candidates"][0].cpu().numpy())
            assert _units(a) == vals.tolist() == out["x"][0].tolist(), i
        else:
            assert svc._exps["svc-a"].engine is None
        rows.append(_units(a))
        losses.append(-_objective(a))

    first, _ = _run(stub, "svc-a", 80, settings, check)
    replica.close()
    again, _ = _run(stub, "svc-b", 80, settings)                 # the same request sequence under another name: same replies
    assert first == again


def test_service_space_change_resets_and_batches(tpe_stub):
    stub, svc = tpe_stub
    settings = {"random_state": 3, "n_startup_jobs": 5}
    _, req = _run(stub, "svc-c", 8, settings)
    st = svc._exps["svc-c"]
    assert len(st.rows) == 7 and st.engine is not None
    req.current_request_number = 3
    rep = stub.GetSuggestions(req)
    pts = [{x.name: x.value for x in pa.assignments} for pa in rep.parameter_assignments]
    assert len(pts) == 3 and len({p["x"] for p in pts}) == 3            # three independent draws against one model
    for p in pts:
        assert -1.0 <= float(p["x"]) < 3.0 and int(p["layers"]) % 5 == 0 and p["opt"] in ("sgd", "adam", "ftrl") and p["bs"] in ("16", "32", "64")
    req.experiment.CopyFrom(_experiment("svc-c", settings, dmax="5.0"))   # same name, wider space: a fresh experiment
    stub.GetSuggestions(req)
    st2 = svc._exps["svc-c"]
    assert st2 is not st and len(st2.rows) == 8 and st.engine is None      # the old engine was closed
