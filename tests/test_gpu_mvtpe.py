"""GPU: the multivariate TPE engine (kbo_mvtpe_*, kubeflow_b200.mvtpe.MvTpe) against its FP64 contract, oracle/mvtpe_oracle.py —
the models it builds, the decision over caller-supplied candidates, its sampler, and the ``multivariate-tpe`` service over
gRPC."""
import grpc
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import mvtpe_oracle as O
from tests import _mvtpe_ref as R

pytestmark = pytest.mark.gpu

KINDS = [("float", -1.0, 3.0), ("int", 0, 19, 1), ("cat", 3), ("int", 3, 48, 5), ("float", 0.0, 1e-3), ("cat", 64)]


def space_of(D):
    return [KINDS[0]] if D == 1 else [KINDS[d % len(KINDS)] for d in range(D)]


def history(space, n, seed):
    """n trials with tied values (a third of every float column on a 0.25-of-range grid) and tied, ±inf losses."""
    r = np.random.default_rng(seed)
    X = np.empty((n, len(space)))
    for d, p in enumerate(space):
        if p[0] == "float":
            v = r.uniform(p[1], p[2], n)
            v[: n // 3] = p[1] + np.round((v[: n // 3] - p[1]) / (p[2] - p[1]) * 4) / 4 * (p[2] - p[1])
        elif p[0] == "int":
            v = O.round_int(p, r.uniform(p[1], p[2], n))
        else:
            v = r.integers(0, p[1], n).astype(float)
        X[:, d] = v
    losses = r.integers(0, max(n // 4, 2), n).astype(float)
    if n > 3:
        losses[1], losses[2] = np.inf, -np.inf
    return X, losses


def engine(space, X, losses, seed=11):
    from kubeflow_b200.mvtpe import MvTpe
    t = MvTpe(space, seed=seed)
    t.tell(X, losses)
    return t


@pytest.mark.parametrize("D", [1, 4, 32, 128])
@pytest.mark.parametrize("n", [1, 2, 9, 10, 11, 250, 251, 8192])
def test_models_match_oracle(n, D):
    space = space_of(D)
    X, losses = history(space, n, seed=n * 1000 + D)
    t = engine(space, X, losses)
    got, ref = t.state(), O.build_models(space, X, losses)
    assert got["n_below"] == ref["n_below"]
    for g in ("below", "above"):
        a, b = got[g], ref[g]
        np.testing.assert_allclose(a["w"], b["w"], rtol=1e-13, atol=0, err_msg=g)
        np.testing.assert_allclose(a["sigma"], b["sigma"], rtol=1e-13, atol=0, equal_nan=True, err_msg=g)
        np.testing.assert_array_equal(a["mu"], b["mu"])
        np.testing.assert_allclose(a["cat_rows"], b["cat_rows"], rtol=1e-13, atol=0, equal_nan=True)
    t.close()


def test_told_values_outside_their_domain_are_refused():
    from kubeflow_b200._lib import KboInvalidArgument
    space = [("float", 0.0, 1.0), ("int", 0, 10, 2), ("cat", 3)]
    t = engine(space, np.zeros((0, 3)), np.zeros(0))
    for row, loss in (([0.5, 2.0, 1.0], np.nan), ([1.5, 2.0, 1.0], 0.0), ([0.5, 3.0, 1.0], 0.0), ([0.5, 2.0, 3.0], 0.0)):
        with pytest.raises(KboInvalidArgument):
            t.tell([row], [loss])
    t.tell([[0.5, 10.0, 2.0]], [np.inf])
    assert t.state()["below"]["mu"].tolist() == [[0.5, 10.0, 2.0]]
    t.close()


SCORING_SPACE = [("float", -1.0, 3.0), ("float", 0.0, 1.0), ("int", 0, 19, 1), ("cat", 5), ("int", 3, 48, 5)]


def _check_decision(space, X, losses, cands, label):
    """Engine on cands (M × D) against the FP64 yardstick: the winner is the first index of the FP64 maximum and every FP32
    score lies within its bound.  Returns the reference scores."""
    M = cands.shape[0]
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    dc = torch.tensor(cands.T[None].copy(), device="cuda")
    out = t.ask(1, M, candidates=dc, return_details=True)
    assert torch.equal(out["candidates"], dc)
    s64 = R.score(space, models, torch.tensor(cands, device="cuda"), chunk=max(64, (1 << 25) // max(len(X), 1))).cpu().numpy()
    if M <= 4096:
        np.testing.assert_allclose(s64, O.score(space, models, cands), rtol=0, atol=1e-10 * (1 + np.abs(s64).max()))
    sc = out["scores"][0].cpu().numpy().astype(np.float64)
    err = np.abs(sc[:, 0] - s64)
    assert (err <= sc[:, 1]).all(), f"{label}: max excess {np.max(err - sc[:, 1]):.3e} at {int(np.argmax(err - sc[:, 1]))}"
    win = int(np.argmax(s64))
    assert int(out["index"][0]) == win, (label, int(out["index"][0]), win, s64[int(out["index"][0])] - s64[win])
    assert out["x"][0].tolist() == cands[win].tolist()
    print(f"\n{label}: survivors {int(out['survivors'][0])}, median bound {np.median(sc[:, 1]):.2e}, max |s32 - s64| {err.max():.2e}, "
          f"max bound / error {np.max(err / sc[:, 1]):.3f}")
    t.close()
    return s64, models


@pytest.mark.parametrize("M", [24, 4096, 1 << 20])
@pytest.mark.parametrize("n", [10, 1000, 8192])
def test_decision_on_supplied_candidates(n, M):
    space = SCORING_SPACE
    X, losses = history(space, n, seed=n + 7)
    models = O.build_models(space, X, losses)
    r = np.random.default_rng(M + n)
    cands = O.draw(space, models, M, r)
    k8 = min(8, n, M)
    cands[:k8] = X[:k8]                                                 # candidates at observed points
    cands[min(8, M - 1), :2] = [-1.0, 0.0]                              # and on the bounds
    cands[min(9, M - 1), :3] = [3.0, 1.0, 19.0]
    if M >= 4096:
        cands[M // 2:] = cands[: M - M // 2]                            # every candidate twice: the first copy must win
    s64, _ = _check_decision(space, X, losses, cands, f"n={n} M={M}")
    if M >= 4096:
        assert int(np.argmax(s64)) < M // 2


WIDE_SPACES = {
    "128 mixed: 43 floats (2 slabs), 85 integers and categoricals (6 slabs)": space_of(128),
    "20 integers and categoricals (2 slabs), no floats": [KINDS[d] for d in (1, 2, 3, 5)] * 5,
    "40 floats (2 slabs), no integers or categoricals": [KINDS[0], KINDS[4], ("float", 2.0, 7.0), ("float", -5.0, -4.0)] * 10,
}


@pytest.mark.parametrize("label", list(WIDE_SPACES))
def test_decision_over_parameter_slabs(label):
    """The score kernel stages float parameters 32 and discrete ones 16 at a time: spaces with several slabs of each, and with
    none of one kind, decide as the FP64 argmax with every FP32 score within its bound."""
    space = WIDE_SPACES[label]
    X, losses = history(space, 1000, seed=len(space))
    models = O.build_models(space, X, losses)
    cands = O.draw(space, models, 4096, np.random.default_rng(len(space) + 1))
    cands[:8] = X[:8]
    cands[2048:] = cands[:2048]
    s64, _ = _check_decision(space, X, losses, cands, label)
    assert int(np.argmax(s64)) < 2048


def test_scores_closer_than_fp32_resolution():
    """Three copies of the best candidate moved by ±1e-9 of the range: FP32 cannot tell them apart, FP64 can."""
    space = SCORING_SPACE
    X, losses = history(space, 1000, seed=3)
    models = O.build_models(space, X, losses)
    cands = O.draw(space, models, 4096, np.random.default_rng(1))
    b = int(np.argmax(O.score(space, models, cands)))
    for i, dx in ((100, -4e-9), (200, 4e-9), (300, 0.0)):
        cands[i] = cands[b]
        cands[i, 0] += dx
    s = O.score(space, models, cands[[100, 200, 300]])
    assert len(set(s.tolist())) == 3 and np.ptp(s) < 1e-6 * abs(s).max()
    _check_decision(space, X, losses, cands, "near ties")


def test_integer_above_the_table_cap():
    """2^18 levels: more than the 2^16 the offset table holds, so every term of that parameter is evaluated in FP64."""
    space = [("float", 0.0, 1.0), ("int", 0, (1 << 18) - 1, 1), ("cat", 4)]
    X, losses = history(space, 1000, seed=21)
    models = O.build_models(space, X, losses)
    cands = O.draw(space, models, 4096, np.random.default_rng(2))
    cands[:5] = X[:5]
    _check_decision(space, X, losses, cands, "int 2^18 levels")


def test_prior_only_model_picks_index_zero():
    """No history (n_startup_trials = 0): both groups are the prior alone, every score is 0 in FP64, every candidate survives to
    the FP64 decision and the first wins."""
    t = engine(SCORING_SPACE, np.zeros((0, 5)), np.zeros(0))
    out = t.ask(2, 4096, return_details=True)
    assert out["index"].tolist() == [0, 0] and out["survivors"].tolist() == [4096, 4096]
    assert (out["scores"][..., 0] == 0).all()
    t.close()


def test_sampler_distribution_joint_and_replay():
    space = [("float", 0.0, 1.0), ("float", 0.0, 1.0), ("int", 3, 48, 5), ("cat", 4)]
    X = np.array([[0.1, 0.1, 3, 0], [0.9, 0.9, 48, 3]] + [[0.5, 0.5, 23, 1]] * 18, dtype=float)
    losses = np.array([0.0, 0.0] + [1.0] * 18)
    t = engine(space, X, losses, seed=2024)
    M = 1 << 20
    out = t.ask(1, M, return_details=True)
    C = out["candidates"][0].cpu().numpy().T
    g = O.build_models(space, X, losses)["below"]
    for d in (0, 1):
        assert (C[:, d] >= 0.0).all() and (C[:, d] <= 1.0).all()
        ks = stats.kstest(C[:, d], lambda x: O.marginal_cdf(space, g, d, x))
        assert ks.statistic < 1.95 / np.sqrt(M), ks
    assert set(np.unique(C[:, 2])) <= set(range(3, 49, 5))
    for d, pmf in ((2, O.int_pmf(space, g, 2)), (3, O.cat_pmf(space, g, 3))):
        key = ((C[:, d] - 3) / 5).astype(int) if d == 2 else C[:, d].astype(int)
        assert stats.chisquare(np.bincount(key, minlength=len(pmf)), pmf * M).pvalue > 1e-3
    off = ((C[:, 0] < 0.5) != (C[:, 1] < 0.5)).mean()
    ref = O.draw(space, O.build_models(space, X, losses), 200_000, np.random.default_rng(0))
    assert abs(off - ((ref[:, 0] < 0.5) != (ref[:, 1] < 0.5)).mean()) < 0.01 and off < 0.3     # independent marginals: 0.5
    t2 = engine(space, X, losses, seed=2024)
    again = t2.ask(1, M, return_details=True)                     # same key (seed, ask 0): bit-identical
    assert torch.equal(again["candidates"], out["candidates"]) and np.array_equal(again["x"], out["x"])
    nxt = t2.ask(1, M, return_details=True)["candidates"]          # next ask counter: new draws
    assert not torch.equal(nxt, out["candidates"])
    t.close()
    t2.close()


# ---- the service over gRPC --------------------------------------------------------------------------------------------------
CATS = ("sgd", "adam", "ftrl")
BS = ("16", "32", "64")


def _experiment(name, settings):
    from kubeflow_b200.suggestion import api_pb as api
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MAXIMIZE
    e.spec.objective.objective_metric_name = "acc"
    e.spec.algorithm.algorithm_name = "multivariate-tpe"
    for k, v in settings.items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, step, lst in (("x", api.DOUBLE, "-1.0", "3.0", "", ()), ("y", api.DOUBLE, "0", "1", "", ()),
                                            ("layers", api.INT, "3", "48", "5", ()), ("opt", api.CATEGORICAL, None, None, "", CATS),
                                            ("bs", api.DISCRETE, None, None, "", BS)):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        if lo is not None:
            p.feasible_space.min, p.feasible_space.max = lo, hi
        if step:
            p.feasible_space.step = step
        p.feasible_space.list.extend(lst)
    return e


def _objective(a):
    return -(float(a["x"]) - 1.3) ** 2 - (float(a["y"]) - float(a["x"]) / 3) ** 2 - 0.01 * abs(int(a["layers"]) - 23) \
        + {"sgd": 0.0, "adam": 0.3, "ftrl": 0.1}[a["opt"]] + 0.001 * int(a["bs"])


def _units(a):
    """A reply in parameter units as the service tells it: start-up points draw every integer in [min, max], and the service
    takes them to the nearest point of the step-5 grid."""
    layers = float(O.round_int(("int", 3, 48, 5), float(a["layers"])))
    return [float(a["x"]), float(a["y"]), layers, float(CATS.index(a["opt"])), float(BS.index(a["bs"]))]


@pytest.fixture(scope="module")
def mv_stub():
    from kubeflow_b200.suggestion.mvtpe_service import MultivariateTpeService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    svc = MultivariateTpeService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


def _run(stub, name, rounds, settings, k, check=None):
    from kubeflow_b200.suggestion import api_pb as api
    exp = _experiment(name, settings)
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=k)
    replies = []
    for i in range(rounds):
        rep = stub.GetSuggestions(req)
        pts = [{x.name: x.value for x in pa.assignments} for pa in rep.parameter_assignments]
        assert len(pts) == k
        replies.append(pts)
        if check:
            check(i, pts)
        for j, a in enumerate(pts):
            t = req.trials.add()
            t.name = f"{name}-t{i}-{j}"
            t.spec.objective.objective_metric_name = "acc"
            for kk, v in a.items():
                x = t.spec.parameter_assignments.assignments.add()
                x.name, x.value = kk, v
            t.status.condition = api.SUCCEEDED
            m = t.status.observation.metrics.add()
            m.name, m.value = "acc", "nan" if (i, j) == (5, 1) else repr(_objective(a))
    return replies


def test_service_rounds_match_oracle_and_replay(mv_stub):
    """64 rounds of 3 points on a mixed 5-D MAXIMIZE space (4 start-up rounds: n_startup_trials = 10).  A replica engine with
    the same seed, history and ask count regenerates the service's candidates; every model-based point equals the oracle's
    choice over them.  The NaN-objective trial of round 5 is never told."""
    from kubeflow_b200.mvtpe import MvTpe
    from kubeflow_b200.suggestion.internal import HyperParameterSearchSpace
    from kubeflow_b200.suggestion.mvtpe_service import mvtpe_space
    stub, svc = mv_stub
    settings = {"random_state": 42, "n_ei_candidates": 64}
    space = mvtpe_space(HyperParameterSearchSpace.convert(_experiment("mv-a", settings)))
    rows, losses = [], []
    replica = MvTpe(space, seed=42)
    told = [0]
    model_rounds = [0]

    def check(i, pts):
        if len(rows) >= 10:
            if told[0] < len(rows):
                replica.tell(np.asarray(rows[told[0]:]), np.asarray(losses[told[0]:]))
                told[0] = len(rows)
            out = replica.ask(3, 64, return_details=True)
            models = O.build_models(space, np.asarray(rows), np.asarray(losses))
            C = out["candidates"].cpu().numpy()
            for j, a in enumerate(pts):
                x, _ = O.choose(space, models, C[j].T)
                assert _units(a) == x.tolist() == out["x"][j].tolist() and int(a["layers"]) % 5 == 3, (i, j)
            model_rounds[0] += 1
        else:
            assert svc._exps["mv-a"].engine is None
        for j, a in enumerate(pts):
            if (i, j) != (5, 1):
                rows.append(_units(a))
                losses.append(-_objective(a))

    first = _run(stub, "mv-a", 64, settings, 3, check)
    replica.close()
    assert model_rounds[0] >= 60 and svc._exps["mv-a"].engine.n == 64 * 3 - 1 - 3      # the last round's points are not told yet
    again = _run(stub, "mv-b", 64, settings, 3)                    # the same request sequence under another name: same replies
    assert first == again
