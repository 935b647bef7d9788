"""CPU: the api.v1.beta1 Suggestion surface through a REAL in-process grpc.server (SURVEY.md §4 item iv):
BASELINE.json config 1 (random search, 4-dim continuous space, 32 trials), ValidateAlgorithmSettings error mapping,
request conversion, both service names, the health endpoint.  The GP algorithm itself needs a GPU: its gRPC test is
in tests/test_gpu_service.py."""
import grpc
import numpy as np
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.internal import AlgorithmSettingsError, HyperParameterSearchSpace, Trial
from kubeflow_b200.suggestion.server import SERVICE_NAMES, SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, RandomService, SkoptService, validate_skopt_settings


def make_experiment(algorithm="random", settings=None, objective=api.MINIMIZE, name="exp-1"):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = objective
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = algorithm
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for i, (lo, hi) in enumerate([(0.01, 0.1), (-1.0, 1.0), (10.0, 20.0), (0.0, 5.0)]):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = f"x{i}", api.DOUBLE
        p.feasible_space.min, p.feasible_space.max = str(lo), str(hi)
    return e


def add_trial(req, name, values, loss, condition=api.SUCCEEDED):
    t = req.trials.add()
    t.name = name
    t.spec.objective.objective_metric_name = "loss"
    for k, v in values.items():
        a = t.spec.parameter_assignments.assignments.add()
        a.name, a.value = k, str(v)
    t.status.condition = condition
    m = t.status.observation.metrics.add()
    m.name, m.value = "loss", str(loss)
    return t


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([SkoptService(), RandomService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def test_config1_random_search_32_trials_over_grpc(stub):
    exp = make_experiment("random", {"random_state": 7})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=4)
    seen = []
    for round_ in range(8):                      # 8 × 4 = 32 trials, each call resends all completed trials
        reply = stub.GetSuggestions(req)
        assert len(reply.parameter_assignments) == 4
        for pa in reply.parameter_assignments:
            vals = {a.name: float(a.value) for a in pa.assignments}
            assert list(vals) == ["x0", "x1", "x2", "x3"]
            for (lo, hi), v in zip([(0.01, 0.1), (-1.0, 1.0), (10.0, 20.0), (0.0, 5.0)], vals.values()):
                assert lo <= v <= hi
            seen.append(tuple(vals.values()))
            add_trial(req, f"t{len(seen)}", vals, loss=sum(vals.values()))
    assert len(seen) == 32 and len(set(seen)) == 32


def test_both_service_names_and_health():
    server, port = serve(RandomService(), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    for name in SERVICE_NAMES:
        s = SuggestionStub(ch, name)
        r = s.GetSuggestions(api.GetSuggestionsRequest(experiment=make_experiment("random"), current_request_number=1))
        assert len(r.parameter_assignments) == 1
    assert SuggestionStub(ch).HealthCheck(b"") == b"\x08\x01"
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("settings,frag", [({"base_estimator": "XGB"}, "base_estimator"), ({"n_initial_points": -1}, "n_initial_points"),
                                            ({"acq_func": "UCBX"}, "acq_func"), ({"acq_optimizer": "adam"}, "acq_optimizer"),
                                            ({"random_state": -3}, "random_state"), ({"n_points": "abc"}, "n_points"),
                                            ({"bogus": 1}, "unknown setting"), ({"kernel": "linear"}, "kernel")])
def test_validate_rejects_bad_settings_with_invalid_argument(stub, settings, frag):
    with pytest.raises(grpc.RpcError) as ei:
        stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment("bayesianoptimization", settings)))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and frag in ei.value.details()


def test_validate_accepts_upstream_and_engine_settings(stub):
    ok = {"base_estimator": "GP", "n_initial_points": 10, "acq_func": "gp_hedge", "acq_optimizer": "auto", "random_state": 1,
          "n_points": 4096, "kernel": "matern52", "noise": 1e-3, "var_mode": "tc"}
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment("bayesianoptimization", ok)))
    assert validate_skopt_settings({k: str(v) for k, v in ok.items()})["n_points"] == 4096


def test_unknown_algorithm_and_bad_space(stub):
    with pytest.raises(grpc.RpcError) as ei:
        stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment("tpe")))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    e = make_experiment("random")
    e.spec.parameter_specs.parameters[0].feasible_space.min = "9"      # min > max
    with pytest.raises(grpc.RpcError) as ei:
        stub.GetSuggestions(api.GetSuggestionsRequest(experiment=e, current_request_number=1))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT


def test_request_conversion_types_and_goal():
    e = make_experiment("random", objective=api.MAXIMIZE)
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "layers", api.INT
    p.feasible_space.min, p.feasible_space.max = "1", "8"
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "opt", api.CATEGORICAL
    p.feasible_space.list.extend(["sgd", "adam", "ftrl"])
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "bs", api.DISCRETE
    p.feasible_space.list.extend(["16", "32"])
    ss = HyperParameterSearchSpace.convert(e)
    assert ss.goal == "MAXIMIZE" and [q.type for q in ss.params] == ["double"] * 4 + ["int", "categorical", "discrete"]
    req = api.GetSuggestionsRequest(experiment=e)
    add_trial(req, "ok", {"x0": 0.05}, 0.5)
    add_trial(req, "running", {"x0": 0.05}, 0.5, condition=1)
    t = req.trials.add(); t.name = "no-metric"; t.status.condition = api.SUCCEEDED
    conv = Trial.convert(req.trials)
    assert [c.name for c in conv] == ["ok"] and conv[0].target_metric.value == "0.5"
    e.spec.objective.type = api.UNKNOWN
    with pytest.raises(AlgorithmSettingsError):
        HyperParameterSearchSpace.convert(e)


def test_space_transform_roundtrip():
    from kubeflow_b200.space import Categorical, Integer, Real, Space
    sp = Space([Real(0.01, 0.1), Integer(1, 8), Categorical(["sgd", "adam", "ftrl"]), Categorical(["16", "32"])])
    assert sp.transformed_n_dims == 1 + 1 + 3 + 1
    pts = [[0.05, 3, "adam", "32"], [0.01, 8, "ftrl", "16"]]
    U = sp.transform(pts)
    assert U.shape == (2, 6) and U.min() >= 0 and U.max() <= 1
    back = sp.inverse_transform(U)
    assert back[0][1:] == [3, "adam", "32"] and abs(back[0][0] - 0.05) < 1e-12 and back[1][1:] == [8, "ftrl", "16"]
    R = sp.rvs_transformed(1000, np.random.default_rng(0))
    assert R.shape == (1000, 6) and np.allclose(R[:, 2:5].sum(1), 1) and set(np.unique(R[:, 5])) == {0.0, 1.0}
    assert np.allclose(R[:, 1] * 7, np.round(R[:, 1] * 7), atol=1e-5)


def test_sobol_is_low_discrepancy_and_resumes():
    """Katib algorithm `sobol`: points stay in bounds, successive calls continue the same sequence, and 64 points cover the
    unit cube more evenly than 64 uniform random points (centred L2 discrepancy)."""
    from scipy.stats import qmc
    from kubeflow_b200.suggestion.service import SobolService
    svc = SobolService()
    exp = make_experiment("sobol", {"random_state": 3}, name="sobol-1")
    svc.validate(exp)
    pts = []
    for k in (16, 16, 32):
        rep = svc.get_suggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=k))
        assert len(rep.parameter_assignments) == k
        pts += [[float(a.value) for a in pa.assignments] for pa in rep.parameter_assignments]
    P = np.asarray(pts)
    lo, hi = np.array([0.01, -1.0, 10.0, 0.0]), np.array([0.1, 1.0, 20.0, 5.0])
    assert (P >= lo).all() and (P <= hi).all() and len({tuple(p) for p in pts}) == 64
    U = (P - lo) / (hi - lo)
    assert qmc.discrepancy(U) < 0.5 * qmc.discrepancy(np.random.default_rng(0).random((64, 4)))
    one = SobolService().get_suggestions(api.GetSuggestionsRequest(experiment=make_experiment("sobol", {"random_state": 3}, name="s2"),
                                                                    current_request_number=64))
    Q = np.asarray([[float(a.value) for a in pa.assignments] for pa in one.parameter_assignments])
    np.testing.assert_allclose(P, Q, rtol=0, atol=1e-12)            # 16 + 16 + 32 == one call of 64


# ---- service state hygiene (round-1 advisor findings) ----------------------------------------------------------------------------
def test_skopt_service_rebuilds_the_optimizer_when_the_experiment_changes():
    """The per-experiment cache is keyed by name AND a fingerprint of (space, objective, settings): an experiment recreated
    under the same name with another space or other settings must not inherit the old optimizer's dimensions or history."""
    svc = SkoptService()
    exp = make_experiment("bayesianoptimization", {"n_initial_points": 50, "random_state": 1})
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=1)
    add_trial(req, "t0", {"x0": 0.05, "x1": 0.0, "x2": 15.0, "x3": 1.0}, 0.3)
    svc.get_suggestions(req)
    first = svc._services["exp-1"]
    assert first.told_trials == {"t0"}
    svc.get_suggestions(req)
    assert svc._services["exp-1"] is first                       # unchanged experiment: same optimizer
    exp2 = make_experiment("bayesianoptimization", {"n_initial_points": 50, "random_state": 1})
    exp2.spec.parameter_specs.parameters[1].feasible_space.max = "3.0"      # same name, wider space
    req2 = api.GetSuggestionsRequest(experiment=exp2, current_request_number=1)
    rep = svc.get_suggestions(req2)
    second = svc._services["exp-1"]
    assert second is not first and second.told_trials == set()
    assert float(second.search_space.params[1].max) == 3.0 and len(rep.parameter_assignments) == 1
    exp3 = make_experiment("bayesianoptimization", {"n_initial_points": 50, "random_state": 2})   # other settings
    svc.get_suggestions(api.GetSuggestionsRequest(experiment=exp3, current_request_number=1))
    assert svc._services["exp-1"] is not second


def test_trials_are_marked_told_only_after_tell_succeeded():
    """A bad later trial (missing assignment) fails the request; the good earlier trial must not be left marked as told
    without having been told — it would be skipped on every later request."""
    svc = SkoptService()
    exp = make_experiment("bayesianoptimization", {"n_initial_points": 50, "random_state": 1}, name="exp-told")
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=1)
    add_trial(req, "good", {"x0": 0.05, "x1": 0.0, "x2": 15.0, "x3": 1.0}, 0.3)
    add_trial(req, "bad", {"x0": 0.05, "x1": 0.0, "x2": 15.0}, 0.4)           # x3 missing
    with pytest.raises(ValueError):
        svc.get_suggestions(req)
    b = svc._services["exp-told"]
    assert b.told_trials == set() and len(b.skopt_optimizer.yi) == 0
    a = req.trials[1].spec.parameter_assignments.assignments.add()
    a.name, a.value = "x3", "2.0"
    svc.get_suggestions(req)
    assert b.told_trials == {"good", "bad"} and len(b.skopt_optimizer.yi) == 2


class _FakeEs:
    """Stand-in for the GPU CMA-ES sampler (kubeflow_b200.cmaes.CmaEs): records tells, hands out fixed populations."""
    def __init__(self, mean0, sigma0, popsize=None, seed=0, device=0):
        self.D, self.popsize, self.told, self.gen = len(mean0), int(popsize or 4), [], 0

    def ask(self):
        class _T:
            def __init__(self, a): self.a = a
            def cpu(self): return self
            def numpy(self): return self.a
        self.gen += 1
        # integer parameter x0 in [0, 3]: samples 0 and 1 round to the same value; sample 3 is clipped at the boundary
        base = np.array([[0.34, 0.2], [0.36, 0.2], [0.9, 0.7], [1.4, 0.7]])
        return _T(np.clip(base + 0.001 * self.gen, 0, 2))

    def tell(self, f):
        self.told.append(np.asarray(f).copy())

    def state(self):
        return {"mean": np.full(self.D, 0.5), "sigma": 0.1, "B": np.eye(self.D), "d": np.ones(self.D)}

    def close(self):
        pass


def test_cmaes_generation_survives_duplicate_assignments_and_failed_trials(monkeypatch):
    import kubeflow_b200.cmaes as cm
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    monkeypatch.setattr(cm, "CmaEs", _FakeEs, raising=False)
    svc = CmaesService()
    e = api.Experiment()
    e.name = "cma-dup"
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "cmaes"
    s = e.spec.algorithm.algorithm_settings.add(); s.name, s.value = "popsize", "4"
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "x0", api.INT
    p.feasible_space.min, p.feasible_space.max = "0", "3"
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "x1", api.DOUBLE
    p.feasible_space.min, p.feasible_space.max = "0", "1"
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=4)
    rep = svc.get_suggestions(req)
    pts = [{a.name: a.value for a in pa.assignments} for pa in rep.parameter_assignments]
    assert pts[0] == pts[1]                                      # two samples, one assignment string
    es = svc._exps["cma-dup"].es
    # results: the duplicates both succeed, sample 2 FAILS, sample 3 succeeds
    add_trial(req, "t0", pts[0], 1.0); add_trial(req, "t1", pts[1], 2.0)
    add_trial(req, "t2", pts[2], 0.0, condition=api.FAILED); add_trial(req, "t3", pts[3], 4.0)
    req.current_request_number = 1
    rep = svc.get_suggestions(req)
    again = {a.name: a.value for a in rep.parameter_assignments[0].assignments}
    assert again == pts[2] and es.told == []                     # the failed sample is handed out again, nothing told yet
    add_trial(req, "t4", again, 3.0)
    rep = svc.get_suggestions(req)
    # samples 2 and 3 share one assignment string too (boundary clip): results are matched to them first-in first-out
    assert len(es.told) == 1 and es.told[0].tolist() == [1.0, 2.0, 4.0, 3.0]   # every sample counted once, by index
    assert es.gen == 2 and len(rep.parameter_assignments) == 1
