"""CPU: `use_separable_cma` on the `cmaes` service: validation over gRPC, and which sampler the service builds (stand-ins
here; tests/test_gpu_sepcma.py runs the real one)."""
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


def _wide(n, settings, name="sep-wide"):
    e = make_experiment("cmaes", settings, name=name)
    del e.spec.parameter_specs.parameters[:]
    for i in range(n):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = f"x{i}", api.DOUBLE
        p.feasible_space.min, p.feasible_space.max = "0", "1"
    return e


@pytest.mark.parametrize("value", ["true", "TRUE", "True", "false", "FALSE", " true "])
def test_use_separable_cma_values(stub, value):
    _validate(stub, make_experiment("cmaes", {"use_separable_cma": value}))


@pytest.mark.parametrize("value", ["yes", "1", "", "on", "truee"])
def test_other_values_are_refused_by_name(stub, value):
    _refused(stub, make_experiment("cmaes", {"use_separable_cma": value}), "use_separable_cma")


@pytest.mark.parametrize("other", ["with_margin", "lr_adapt"])
def test_beside_with_margin_or_lr_adapt_is_refused_naming_both(stub, other):
    _refused(stub, make_experiment("cmaes", {"use_separable_cma": "true", other: "true"}), "use_separable_cma", other)


@pytest.mark.parametrize("other", ["with_margin", "lr_adapt"])
def test_off_beside_with_margin_or_lr_adapt_is_accepted(stub, other):
    _validate(stub, make_experiment("cmaes", {"use_separable_cma": "false", other: "true"}))
    _validate(stub, make_experiment("cmaes", {"use_separable_cma": "true", other: "false"}))


def test_with_margin_and_lr_adapt_error_texts_are_unchanged(stub):
    _refused(stub, make_experiment("cmaes", {"with_margin": "yes"}), "failed to convert 'yes' for setting with_margin")
    _refused(stub, make_experiment("cmaes", {"lr_adapt": "yes"}), "failed to convert 'yes' for setting lr_adapt")
    _refused(stub, make_experiment("cmaes", {"lr_adapt": "true", "with_margin": "true"}),
             "lr_adapt: true cannot be combined with with_margin: true")


@pytest.mark.parametrize("settings", [{"restart_strategy": "ipop"}, {"restart_strategy": "bipop"}, {"popsize": "32", "sigma": "0.3"},
                                      {"restart_strategy": "bipop", "popsize": "12", "sigma": "0.2", "random_state": "4"}])
def test_works_with_the_other_settings(stub, settings):
    _validate(stub, make_experiment("cmaes", {"use_separable_cma": "true", **settings}))


def test_4096_parameters_are_accepted_and_4097_refused(stub):
    _validate(stub, _wide(4096, {"use_separable_cma": "true"}))
    _refused(stub, _wide(4097, {"use_separable_cma": "true"}), "use_separable_cma", "4096", "4097")


class _SepEs(_FlagEs):
    """Stand-in for both samplers that records which one the service built."""
    made = []

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.closed = False
        _SepEs.made.append(self)

    def close(self):
        self.closed = True


class _Full(_SepEs):
    sep = False


class _Sep(_SepEs):
    sep = True


def test_toggling_use_separable_cma_starts_a_new_run(monkeypatch):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _Full, raising=False)
    monkeypatch.setattr(cm, "SepCmaEs", _Sep, raising=False)
    svc = CmaesService()
    runs = []
    for value in (None, "true", "TRUE", "false", "true"):
        e = make_experiment("cmaes", {} if value is None else {"use_separable_cma": value}, name="sep-toggle")
        svc.get_suggestions(api.GetSuggestionsRequest(experiment=e, current_request_number=2))
        runs.append(svc._exps["sep-toggle"].es)
    a, b, b2, c, d = runs
    assert b is b2                                   # the same setting keeps its sampler
    assert len({id(a), id(b), id(c), id(d)}) == 4     # every change of the setting starts a new run
    assert (a.sep, b.sep, c.sep, d.sep) == (False, True, False, True)
    assert a.closed and b.closed and c.closed and not d.closed


def test_exhausted_generation_draws_from_the_diagonal(monkeypatch):
    import numpy as np

    import kubeflow_b200.cmaes as cm

    class _Diag(_Sep):
        def state(self):                              # no basis B: the extra draw is mean + σ·(d∘z)
            return {"mean": np.full(self.D, 0.5), "sigma": 0.1, "d": np.linspace(0.5, 2.0, self.D)}
    monkeypatch.setattr(cm, "SepCmaEs", _Diag, raising=False)
    svc = CmaesService()
    e = _wide(300, {"use_separable_cma": "true", "popsize": "4"}, name="sep-extra")
    rep = svc.get_suggestions(api.GetSuggestionsRequest(experiment=e, current_request_number=7))
    assert len(rep.parameter_assignments) == 7
    for pa in rep.parameter_assignments:
        assert all(0.0 <= float(x.value) <= 1.0 for x in pa.assignments)
