"""CPU: `restart_strategy` on the `cmaes` service with a stand-in sampler whose termination flags fire at chosen
generations: validation over gRPC, restarts at exactly those generations with the schedule's λ, σ and mean, no flag read
without a strategy, and the per-sample bookkeeping (duplicates, failed trials) across a restart."""
import grpc
import numpy as np
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.cma_restart import Schedule
from kubeflow_b200.suggestion.cmaes_service import CmaesService
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService
from tests.test_grpc_service import add_trial, make_experiment


class _T:
    def __init__(self, a): self.a = a
    def cpu(self): return self
    def numpy(self): return self.a


class _FlagEs:
    """Stand-in for kubeflow_b200.cmaes.CmaEs: distinct points, stop flags set after the tells listed in `fire_at`."""
    fire_at, last = set(), None

    def __init__(self, mean0, sigma0, popsize=None, seed=0, device=0):
        self.D = len(mean0)
        self.popsize = int(popsize or 4 + int(3 * np.log(self.D)))
        self.tells, self.flag_reads, self.restarts, self.asks = [], 0, [], 0
        self.r = np.random.default_rng(seed)
        _FlagEs.last = self

    def ask(self):
        self.asks += 1
        return _T(self.r.uniform(0.05, 0.95, (self.popsize, self.D)))

    def tell(self, f):
        assert len(f) == self.popsize
        self.tells.append(np.asarray(f).copy())

    def stop_flags(self):
        self.flag_reads += 1
        return (2 if len(self.tells) in self.fire_at else 0), np.zeros(2), 1

    def restart(self, popsize, mean, sigma):
        self.restarts.append((len(self.tells), popsize, np.asarray(mean).copy(), sigma))
        self.popsize = popsize

    def state(self):
        return {"mean": np.full(self.D, 0.5), "sigma": 0.1, "B": np.eye(self.D), "d": np.ones(self.D)}

    def close(self):
        pass


@pytest.fixture
def fake(monkeypatch):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _FlagEs, raising=False)
    return _FlagEs


def _drive(svc, exp, generations):
    """Complete `generations` generations: fetch the generation's points, report a loss for each, let the next call tell."""
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=0)
    svc.get_suggestions(req)
    k = 0
    for _ in range(generations):
        st = svc._exps[exp.name]
        req.current_request_number = len(st.queue)
        rep = svc.get_suggestions(req)
        for pa in rep.parameter_assignments:
            pt = {a.name: a.value for a in pa.assignments}
            add_trial(req, f"t{k}", pt, float(sum(float(v) for v in pt.values())))
            k += 1
        req.current_request_number = 0
        svc.get_suggestions(req)                       # tells the generation (and restarts if a flag is set)
    return svc._exps[exp.name]


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([CmaesService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("value", ["none", "ipop", "bipop"])
def test_accepted_values(stub, value):
    exp = make_experiment("cmaes", {"restart_strategy": value})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))


@pytest.mark.parametrize("value", ["foo", "IPOP", ""])
def test_other_values_are_invalid_argument(stub, value):
    exp = make_experiment("cmaes", {"restart_strategy": value})
    with pytest.raises(grpc.RpcError) as e:
        stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    assert e.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    assert "restart_strategy" in e.value.details() and "none, ipop, bipop" in e.value.details()


@pytest.mark.parametrize("strategy,settings", [("ipop", {}), ("bipop", {"popsize": 5, "sigma": 0.3, "random_state": 9})])
def test_restarts_at_the_flagged_generations_on_the_schedule(fake, strategy, settings):
    fake.fire_at = {3, 7, 8, 12}
    svc = CmaesService()
    exp = make_experiment("cmaes", {"restart_strategy": strategy, **settings}, name=f"cma-{strategy}")
    st = _drive(svc, exp, 14)
    es = fake.last
    assert len(es.tells) == 14 and es.flag_reads == 14
    ref = Schedule(strategy, 4, settings.get("popsize"), settings.get("sigma", 1.0 / 6.0), settings.get("random_state", 0))
    lam, start = ref.lam0, 0
    for (at, got_lam, got_mean, got_sigma), stop in zip(es.restarts, sorted(fake.fire_at)):
        assert at == stop
        assert all(len(f) == lam for f in es.tells[start:stop])           # every tell of the run had that run's λ
        want_lam, want_mean, want_sigma = ref.next_run(lam, stop - start)
        assert (got_lam, got_sigma) == (want_lam, want_sigma) and np.array_equal(got_mean, want_mean)
        lam, start = want_lam, stop
    assert len(es.restarts) == 4 and st.run_gens == 2
    assert all(len(f) == lam for f in es.tells[start:])


@pytest.mark.parametrize("settings", [{}, {"restart_strategy": "none"}])
def test_without_a_strategy_the_flags_are_never_read(fake, settings):
    fake.fire_at = {1, 2, 3}
    svc = CmaesService()
    _drive(svc, make_experiment("cmaes", settings, name="cma-none"), 4)
    es = fake.last
    assert len(es.tells) == 4 and es.flag_reads == 0 and es.restarts == []


class _DupEs(_FlagEs):
    """The fixed populations of test_cmaes_generation_survives…: two samples round to one integer value, two clip to
    the same boundary point.  Rows past the fourth (a larger population after a restart) are distinct."""

    def ask(self):
        self.asks += 1
        base = np.array([[0.34, 0.2], [0.36, 0.2], [0.9, 0.7], [1.4, 0.7]])
        extra = np.column_stack([np.full(self.popsize - 4, 0.5), np.linspace(0.3, 0.6, self.popsize - 4)])
        return _T(np.clip(np.vstack([base + 0.001 * self.asks, extra]), 0, 2))


def test_duplicates_and_failed_trials_across_a_restart(monkeypatch):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _DupEs, raising=False)
    _DupEs.fire_at = {1}
    svc = CmaesService()
    e = api.Experiment()
    e.name = "cma-dup-restart"
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "cmaes"
    for k, v in (("popsize", "4"), ("restart_strategy", "ipop")):
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, v
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "x0", api.INT
    p.feasible_space.min, p.feasible_space.max = "0", "3"
    p = e.spec.parameter_specs.parameters.add(); p.name, p.parameter_type = "x1", api.DOUBLE
    p.feasible_space.min, p.feasible_space.max = "0", "1"
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=4)
    rep = svc.get_suggestions(req)
    pts = [{a.name: a.value for a in pa.assignments} for pa in rep.parameter_assignments]
    for i, pt in enumerate(pts):
        add_trial(req, f"a{i}", pt, float(i))
    req.current_request_number = 8                          # tells generation 1; its flag restarts at λ = 8
    rep = svc.get_suggestions(req)
    es = _DupEs.last
    assert len(es.tells) == 1 and [r[:2] for r in es.restarts] == [(1, 8)] and es.popsize == 8
    pts = [{a.name: a.value for a in pa.assignments} for pa in rep.parameter_assignments]
    assert len(pts) == 8 and pts[0] == pts[1]                   # two samples, one assignment string
    # the duplicates both succeed, sample 2 FAILS, the rest succeed
    for i, pt in enumerate(pts):
        add_trial(req, f"b{i}", pt, 0.0 if i == 2 else 10.0 + i, condition=api.FAILED if i == 2 else api.SUCCEEDED)
    req.current_request_number = 1
    rep = svc.get_suggestions(req)
    again = {a.name: a.value for a in rep.parameter_assignments[0].assignments}
    assert again == pts[2] and len(es.tells) == 1               # the failed sample is handed out again
    add_trial(req, "b8", again, 3.0)
    rep = svc.get_suggestions(req)
    # samples 2 and 3 share one assignment string (boundary clip): matched first-in first-out, every sample once, by index
    assert len(es.tells) == 2 and es.tells[1].tolist() == [10.0, 11.0, 13.0, 3.0, 14.0, 15.0, 16.0, 17.0]
    assert len(rep.parameter_assignments) == 1 and es.flag_reads == 2
