"""CPU: `with_margin` and `margin` on the `cmaes` service: validation over gRPC, and what the service hands the sampler
(a stand-in here; tests/test_gpu_cma_margin.py runs the real one)."""
import grpc
import numpy as np
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.cmaes_service import CmaesService
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService
from tests.test_cmaes_restart_service import _FlagEs, _T
from tests.test_grpc_service import make_experiment


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([CmaesService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _add(e, name, kind, lo=None, hi=None, step=None, values=None):
    p = e.spec.parameter_specs.parameters.add()
    p.name, p.parameter_type = name, kind
    if values is not None:
        p.feasible_space.list.extend(values)
    else:
        p.feasible_space.min, p.feasible_space.max = lo, hi
        if step:
            p.feasible_space.step = step
    return e


def _validate(stub, exp):
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))


def _refused(stub, exp, *words):
    with pytest.raises(grpc.RpcError) as e:
        _validate(stub, exp)
    assert e.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    for w in words:
        assert w in e.value.details(), e.value.details()


@pytest.mark.parametrize("value", ["true", "TRUE", "False", "false"])
def test_with_margin_values(stub, value):
    _validate(stub, make_experiment("cmaes", {"with_margin": value}))


@pytest.mark.parametrize("value", ["yes", "1", "", "truee"])
def test_other_with_margin_values_are_refused(stub, value):
    _refused(stub, make_experiment("cmaes", {"with_margin": value}), "with_margin")


@pytest.mark.parametrize("value", ["0", "1", "-0.1", "1.5", "abc", "nan"])
def test_margin_out_of_range_is_refused(stub, value):
    _refused(stub, make_experiment("cmaes", {"with_margin": "true", "margin": value}), "margin")


def test_margin_in_range_is_accepted(stub):
    _validate(stub, make_experiment("cmaes", {"with_margin": "true", "margin": "0.05"}))


@pytest.mark.parametrize("settings", [{}, {"with_margin": "false"}])
def test_margin_without_with_margin_is_refused_by_name(stub, settings):
    _refused(stub, make_experiment("cmaes", {**settings, "margin": "0.1"}), "margin", "with_margin")


def test_discrete_only_under_with_margin(stub):
    mk = lambda s: _add(make_experiment("cmaes", s), "d", api.DISCRETE, values=["1", "2", "8"])
    _refused(stub, mk({}), "categorical/discrete", "'d'")
    _refused(stub, mk({"with_margin": "false"}), "categorical/discrete")
    _validate(stub, mk({"with_margin": "true"}))
    bad = _add(make_experiment("cmaes", {"with_margin": "true"}), "d", api.DISCRETE, values=["a", "b"])
    _refused(stub, bad, "'d'", "numeric")


@pytest.mark.parametrize("settings", [{}, {"with_margin": "true"}])
def test_int_accepted_and_categorical_still_refused(stub, settings):
    _validate(stub, _add(make_experiment("cmaes", settings), "n", api.INT, "1", "8", "2"))
    _refused(stub, _add(make_experiment("cmaes", settings), "c", api.CATEGORICAL, values=["a", "b"]),
             "categorical/discrete", "'c'")


class _MarginEs(_FlagEs):
    """Stand-in that records set_margin and samples the levels it was given."""

    def set_margin(self, dims, alpha=None):
        self.margin = (dims, alpha)

    def ask(self):
        X = self.r.uniform(0.05, 0.95, (self.popsize, self.D))
        for j, c in self.margin[0].items():
            X[:, j] = self.r.choice(np.asarray(c), self.popsize)
        return _T(X)


@pytest.mark.parametrize("alpha", [None, 0.2])
def test_service_hands_the_levels_to_the_sampler_and_their_values_to_trials(monkeypatch, alpha):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _MarginEs, raising=False)
    s = {"with_margin": "true", **({"margin": alpha} if alpha else {})}
    e = make_experiment("cmaes", s, name=f"margin-{alpha}")
    _add(e, "n", api.INT, "2", "11", "3")
    _add(e, "d", api.DISCRETE, values=["0.5", "16", "4"])
    svc = CmaesService()
    rep = svc.get_suggestions(api.GetSuggestionsRequest(experiment=e, current_request_number=8))
    es = _MarginEs.last
    dims, got_alpha = es.margin
    assert sorted(dims) == [4, 5] and got_alpha == alpha
    assert np.allclose(dims[4], [0, 1 / 3, 2 / 3, 1]) and np.allclose(dims[5], [0, 3.5 / 15.5, 1])
    for pa in rep.parameter_assignments:
        a = {x.name: x.value for x in pa.assignments}
        assert a["n"] in ("2", "5", "8", "11") and a["d"] in ("0.5", "4", "16")
