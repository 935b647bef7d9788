"""CPU: the ``tpe`` service's settings validation over a real gRPC server, and its start-up phase, which needs no CUDA device
(the model-based phase is tested on the GPU in tests/test_gpu_tpe.py)."""
import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService
from kubeflow_b200.suggestion.tpe_service import TpeService, validate_tpe_settings


def make_experiment(settings=None, name="tpe-1"):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "tpe"
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, step, lst in (("lr", api.DOUBLE, "0.001", "0.1", "", ()), ("layers", api.INT, "2", "12", "2", ()),
                                            ("opt", api.CATEGORICAL, None, None, "", ("sgd", "adam")),
                                            ("bs", api.DISCRETE, None, None, "", ("16", "32", "64"))):
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
    svc = TpeService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("name,value", [("gamma", 0), ("gamma", 1), ("gamma", "x"), ("prior_weight", 0), ("prior_weight", -1),
                                        ("n_EI_candidates", 0), ("n_EI_candidates", 1 << 25), ("n_startup_jobs", -1),
                                        ("random_state", -2), ("device", -1), ("bogus", 1)])
def test_bad_settings_give_invalid_argument_naming_the_setting(stub, name, value):
    with pytest.raises(grpc.RpcError) as ei:
        stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment({name: value})))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and name in ei.value.details()


def test_good_settings_validate(stub):
    ok = {"gamma": 0.3, "prior_weight": 2.0, "n_EI_candidates": 4096, "n_startup_jobs": 0, "random_state": 7, "device": 0}
    stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(ok)))
    got = validate_tpe_settings({k: str(v) for k, v in ok.items()})
    assert got["gamma"] == 0.3 and got["n_EI_candidates"] == 4096 and got["n_startup_jobs"] == 0
    assert validate_tpe_settings({}) == dict(gamma=0.25, prior_weight=1.0, n_EI_candidates=24, n_startup_jobs=20)


def test_startup_phase_needs_no_device_and_stays_in_bounds(stub):
    s, svc = stub
    req = api.GetSuggestionsRequest(experiment=make_experiment({"random_state": 5}, name="tpe-start"), current_request_number=4)
    for r in range(4):                                        # 16 points, all before n_startup_jobs = 20 trials are told
        rep = s.GetSuggestions(req)
        assert len(rep.parameter_assignments) == 4
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
            m.name, m.value = "loss", "0.5"
    st = svc._exps["tpe-start"]
    assert st.engine is None and len(st.rows) == 12 and st.rows[0][2] in (0.0, 1.0)


def test_bad_trial_value_is_invalid_argument_and_nothing_is_told(stub):
    s, svc = stub
    req = api.GetSuggestionsRequest(experiment=make_experiment({}, name="tpe-bad"), current_request_number=1)
    for name, opt in (("good", "sgd"), ("bad", "rmsprop")):
        t = req.trials.add()
        t.name = name
        t.spec.objective.objective_metric_name = "loss"
        for k, v in (("lr", "0.01"), ("layers", "4"), ("opt", opt), ("bs", "32")):
            x = t.spec.parameter_assignments.assignments.add()
            x.name, x.value = k, v
        t.status.condition = api.SUCCEEDED
        m = t.status.observation.metrics.add()
        m.name, m.value = "loss", "1.0"
    with pytest.raises(grpc.RpcError) as ei:
        s.GetSuggestions(req)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and "rmsprop" in ei.value.details()
    assert svc._exps["tpe-bad"].told == set()
