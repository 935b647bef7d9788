"""CPU: ValidateAlgorithmSettings of ``bayesianoptimization`` with the tree estimators, over a real in-process gRPC server."""
import grpc
import pytest

from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Real
from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, SkoptService
from tests.test_grpc_service import make_experiment


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([SkoptService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _validate(stub, settings):
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment("bayesianoptimization", settings)))


@pytest.mark.parametrize("est", ["RF", "ET"])
def test_tree_estimators_are_accepted(stub, est):
    _validate(stub, {"base_estimator": est, "n_initial_points": 5, "acq_func": "gp_hedge", "acq_optimizer": "auto", "random_state": 3,
                     "n_points": 4096, "xi": 0.02, "kappa": 2.5, "candidate_backend": "numpy"})
    _validate(stub, {"base_estimator": est, "acq_optimizer": "sampling", "acq_func": "EI"})


@pytest.mark.parametrize("est", ["GBRT", "XGB"])
def test_other_estimators_stay_refused(stub, est):
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, {"base_estimator": est})
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and f"base_estimator {est}" in ei.value.details()


@pytest.mark.parametrize("est,cls", [("RF", "RandomForestRegressor"), ("ET", "ExtraTreesRegressor")])
def test_lbfgs_with_a_tree_estimator_is_refused_in_skopt_words(stub, est, cls):
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, {"base_estimator": est, "acq_optimizer": "lbfgs"})
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    assert ei.value.details() == f"The regressor {cls} should run with acq_optimizer='sampling'."
    with pytest.raises(ValueError, match="should run with acq_optimizer='sampling'"):
        Optimizer([Real(0.0, 1.0)], base_estimator=est, acq_optimizer="lbfgs")


@pytest.mark.parametrize("knob,value", [("kernel", "rbf"), ("length_scale", 0.5), ("amplitude", 2.0), ("noise", 1e-4), ("var_mode", "tc"),
                                        ("theta_grid", 3), ("theta_search", 2), ("theta_fit", "lbfgs"), ("ard", 1)])
def test_gp_only_knobs_are_refused_with_a_tree_estimator(stub, knob, value):
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, {"base_estimator": "RF", knob: value})
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and knob in ei.value.details()
    _validate(stub, {"base_estimator": "GP", knob: value})        # still fine for the GP


def test_optimizer_refuses_gbrt_without_touching_a_device():
    with pytest.raises(ValueError, match="GBRT"):
        Optimizer([Real(0.0, 1.0)], base_estimator="GBRT")
    opt = Optimizer([Real(0.0, 1.0)], base_estimator="ET", n_initial_points=3, random_state=0)
    assert opt.forest and opt._engine is None
    assert len(opt.ask(n_points=2)) == 2                          # the random start-up phase needs no device
