"""CPU: `lr_adapt` on the `cmaes` service: validation over gRPC, and what the service hands the sampler (a stand-in here;
tests/test_gpu_cma_lra.py runs the real one)."""
import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.cmaes_service import CmaesService
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService
from tests.test_cmaes_margin_service import _refused, _validate
from tests.test_cmaes_restart_service import _FlagEs
from tests.test_grpc_service import make_experiment


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([CmaesService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("value", ["true", "TRUE", "True", "false", "FALSE", " false "])
def test_lr_adapt_values(stub, value):
    _validate(stub, make_experiment("cmaes", {"lr_adapt": value}))


@pytest.mark.parametrize("value", ["yes", "1", "", "on", "truee"])
def test_other_lr_adapt_values_are_refused_by_name(stub, value):
    _refused(stub, make_experiment("cmaes", {"lr_adapt": value}), "lr_adapt")


def test_with_margin_error_text_is_unchanged(stub):
    _refused(stub, make_experiment("cmaes", {"with_margin": "yes"}), "failed to convert 'yes' for setting with_margin")


def test_lr_adapt_beside_with_margin_is_refused_naming_both(stub):
    _refused(stub, make_experiment("cmaes", {"lr_adapt": "true", "with_margin": "true"}), "lr_adapt", "with_margin")


@pytest.mark.parametrize("settings", [{"with_margin": "false"}, {"restart_strategy": "ipop"}, {"restart_strategy": "bipop"},
                                      {"popsize": "32", "sigma": "0.3"},
                                      {"restart_strategy": "bipop", "popsize": "12", "sigma": "0.2", "random_state": "4"}])
def test_lr_adapt_works_with_the_other_settings(stub, settings):
    _validate(stub, make_experiment("cmaes", {"lr_adapt": "true", **settings}))


class _LraEs(_FlagEs):
    """Stand-in that records set_lr_adapt."""
    made = []

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.lr_adapt = None
        self.closed = False
        _LraEs.made.append(self)

    def set_lr_adapt(self, on):
        self.lr_adapt = on

    def close(self):
        self.closed = True


def test_toggling_lr_adapt_starts_a_new_run(monkeypatch):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _LraEs, raising=False)
    _LraEs.made = []
    svc = CmaesService()
    runs = []
    for value in (None, "true", "true", "false", "TRUE"):
        e = make_experiment("cmaes", {} if value is None else {"lr_adapt": value}, name="lra-toggle")
        svc.get_suggestions(api.GetSuggestionsRequest(experiment=e, current_request_number=2))
        runs.append(svc._exps["lra-toggle"].es)
    a, b, b2, c, d = runs
    assert b is b2                                   # the same setting keeps its sampler
    assert len({id(a), id(b), id(c), id(d)}) == 4     # every change of the setting starts a new run
    assert (a.lr_adapt, b.lr_adapt, c.lr_adapt, d.lr_adapt) == (None, True, None, True)
    assert a.closed and b.closed and c.closed and not d.closed
