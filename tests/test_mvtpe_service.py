"""CPU: the ``multivariate-tpe`` service's settings validation over a real gRPC server, its start-up phase with the GPU engine
unimportable, and routing through DispatchService (the model-based phase is tested on the GPU in tests/test_gpu_mvtpe.py)."""
import builtins

import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.mvtpe_service import MAX_PARAMETERS, MultivariateTpeService, validate_mvtpe_settings
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, RandomService
from kubeflow_b200.suggestion.tpe_service import TpeService

PARAMS = (("lr", api.DOUBLE, "0.001", "0.1", "", ()), ("layers", api.INT, "2", "12", "2", ()),
          ("opt", api.CATEGORICAL, None, None, "", ("sgd", "adam")), ("bs", api.DISCRETE, None, None, "", ("16", "32", "64")))


def make_experiment(settings=None, name="mvtpe-1", algorithm="multivariate-tpe", params=PARAMS):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = algorithm
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, step, lst in params:
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        if lo is not None:
            p.feasible_space.min, p.feasible_space.max = lo, hi
        if step:
            p.feasible_space.step = step
        p.feasible_space.list.extend(lst)
    return e


@pytest.fixture(scope="module")
def stub():
    svc = MultivariateTpeService()
    server, port = serve(DispatchService([RandomService(), TpeService(), svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("name,value", [("n_startup_trials", -1), ("n_startup_trials", "x"), ("n_ei_candidates", 0),
                                        ("n_ei_candidates", (1 << 24) + 1), ("n_ei_candidates", "1.5"), ("random_state", -2),
                                        ("random_state", "seed"), ("device", -1), ("gamma", 0.25), ("bogus", 1)])
def test_bad_settings_give_invalid_argument_naming_the_setting(stub, name, value):
    with pytest.raises(grpc.RpcError) as ei:
        stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment({name: value})))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and name in ei.value.details()


def test_good_settings_validate(stub):
    ok = {"n_startup_trials": 0, "n_ei_candidates": 1 << 24, "random_state": 7, "device": 0}
    stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(ok)))
    assert validate_mvtpe_settings({k: str(v) for k, v in ok.items()}) == ok
    assert validate_mvtpe_settings({}) == dict(n_startup_trials=10, n_ei_candidates=24)


def test_space_limits_are_invalid_argument(stub):
    wide = tuple((f"p{i}", api.DOUBLE, "0", "1", "", ()) for i in range(MAX_PARAMETERS + 1))
    for params, needle in ((wide, str(MAX_PARAMETERS)), ((("x", api.DOUBLE, "1", "1", "", ()),), "min < max")):
        with pytest.raises(grpc.RpcError) as ei:
            stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(params=params)))
        assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and needle in ei.value.details()


def test_startup_phase_needs_no_device_and_stays_in_bounds(stub, monkeypatch):
    real_import = builtins.__import__

    def no_engine(name, *a, **kw):
        if name.endswith("mvtpe") and "service" not in name:
            raise ImportError("the GPU engine is not importable in this test")
        return real_import(name, *a, **kw)

    monkeypatch.setattr(builtins, "__import__", no_engine)
    s, svc = stub
    req = api.GetSuggestionsRequest(experiment=make_experiment({"random_state": 5, "n_startup_trials": 12}, name="mv-start"),
                                    current_request_number=3)
    for r in range(4):                                        # 12 points, all before n_startup_trials = 12 trials are told
        rep = s.GetSuggestions(req)
        assert len(rep.parameter_assignments) == 3
        for i, pa in enumerate(rep.parameter_assignments):
            a = {x.name: x.value for x in pa.assignments}
            assert list(a) == ["lr", "layers", "opt", "bs"]
            assert 0.001 <= float(a["lr"]) <= 0.1 and a["layers"] == str(int(a["layers"])) and 2 <= int(a["layers"]) <= 12
            assert a["opt"] in ("sgd", "adam") and a["bs"] in ("16", "32", "64")
            t = req.trials.add()
            t.name = f"t{r}-{i}"
            t.spec.objective.objective_metric_name = "loss"
            for k, v in a.items():
                x = t.spec.parameter_assignments.assignments.add()
                x.name, x.value = k, v
            t.status.condition = api.SUCCEEDED
            m = t.status.observation.metrics.add()
            m.name, m.value = "loss", "nan" if (r, i) == (0, 0) else "0.5"
    st = svc._exps["mv-start"]
    assert st.engine is None and len(st.rows) == 8 and len(st.told) == 9    # the NaN-objective trial is never told
    assert all(row[1] in (2.0, 4.0, 6.0, 8.0, 10.0, 12.0) for row in st.rows)     # integers on the step-2 grid


def test_routing_through_dispatch(stub):
    s, svc = stub
    rep = s.GetSuggestions(api.GetSuggestionsRequest(experiment=make_experiment({"random_state": 1}, name="mv-route"),
                                                     current_request_number=2))
    assert len(rep.parameter_assignments) == 2 and "mv-route" in svc._exps
    with pytest.raises(grpc.RpcError) as ei:
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(algorithm="multivariate-tpe2")))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and "multivariate-tpe2" in ei.value.details()
    with pytest.raises(grpc.RpcError) as ei:                 # the same settings under tpe are tpe's to judge
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment({"n_ei_candidates": 8}, algorithm="tpe")))
    assert "n_ei_candidates" in ei.value.details()
