"""GPU: the CMA-ES termination test (cma_stop_kernel), restart in place (kbo_cma_restart) and the `cmaes` service's IPOP /
BIPOP restarts.

* Criteria: after every tell of every run here, the GPU's flags equal `cma_restart_oracle.should_stop` evaluated on the
  GPU's own exported state (mean, σ, C, p_c, B, d, generation) and history, and the history equals each generation's best
  and worst fitness (NaN and ±inf fitness included).  Over the runs of this file every one of the six bits fires.
* Restart in place equals a fresh instance bit for bit, and the built-in sampler never repeats an earlier draw.
* Without a restart, 200 generations at (D = 128, λ = 4096) and (D = 10, λ = 10) reproduce the parent commit's arithmetic
  bit for bit (SHA-256 of X and the state, generated with the parent commit's library on an H100).
* IPOP and BIPOP runs on rotated Rastrigin pass the resynchronised per-generation check of test_gpu_cma_long.py.
* gRPC Experiments with `restart_strategy` ipop / bipop restart on the schedule.
"""
import importlib.util
import os

import grpc
import numpy as np
import pytest
import torch

from oracle import cma_oracle as O
from oracle import cma_restart_oracle as R
from tests.test_gpu_cma_long import LIMITS, TOL_PS, _errors, _load, _philox_normals

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
SEEN = set()          # bits seen firing over the module
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _es(D, lam, seed=0, mean=0.5, sigma=1.0 / 6.0):
    from kubeflow_b200.cmaes import CmaEs
    return CmaEs(np.full(D, mean) if np.isscalar(mean) else mean, sigma, popsize=lam, seed=seed)


class Checker:
    """Follows one CmaEs: after every tell, the GPU history against a host ring and the GPU flags against the oracle."""

    def __init__(self, es, sigma0):
        self.es = es
        self.start(sigma0)

    def start(self, sigma0):
        self.tolx = R.tolx(sigma0)
        self.term = R.funhist_term(self.es.D, self.es.popsize)
        self.hist = np.zeros(2 * self.term)
        flags, hist, term = self.es.stop_flags()
        assert flags == 0 and term == self.term and not hist.any()

    def after_tell(self, f):
        st = self.es.state()
        g = st["generation"]
        R.record(self.hist, g, self.term, f)
        flags, hist, term = self.es.stop_flags()
        assert term == self.term and np.array_equal(hist, self.hist, equal_nan=True), g
        want = R.should_stop(st["mean"], st["sigma"], st["C"], st["pc"], st["B"], st["d"], hist, g, term, self.tolx)
        assert flags == want, f"generation {g}: GPU flags {flags:#x}, oracle on the GPU state {want:#x}"
        SEEN.update(b for b, v in R.BITS.items() if flags & v)
        return flags


def _drive(D, lam, f, gens, mean=0.5, sigma=1.0 / 6.0, seed=0, until=None):
    es = _es(D, lam, seed, mean, sigma)
    ck = Checker(es, sigma)
    seen = 0
    for _ in range(gens):
        fx = f(es.ask().cpu().numpy())
        es.tell(fx)
        fl = ck.after_tell(fx)
        seen |= fl
        if until is not None and fl & until:
            break
    es.close()
    return seen


def test_tolxup_from_a_huge_sigma():
    assert _drive(4, 8, O.sphere, 3, sigma=1e5) & R.TOLXUP


def test_noeffect_coord_and_axis_at_mean_1e17():
    seen = _drive(4, 8, lambda X: ((X - 1e17) ** 2).sum(1), 5, mean=1e17)
    assert seen & R.NOEFFECTCOORD and seen & R.NOEFFECTAXIS


def test_tolfun_on_constant_fitness():
    D, lam = 3, 7
    term = R.funhist_term(D, lam)
    seen = _drive(D, lam, lambda X: np.full(len(X), 2.5), term + 1)
    assert seen & R.TOLFUN


def test_tolx_on_a_long_sphere_run():
    xs = np.array([0.3, 0.6])
    assert _drive(2, 6, lambda X: 1e20 * ((X - xs) ** 2).sum(1), 1000, until=R.TOLX) & R.TOLX


def test_conditioncov_on_an_ill_conditioned_ellipsoid():
    s, xe = np.array([1.0, 1e28]), np.array([0.3, 0.0])
    assert _drive(2, 6, lambda X: (((X - xe) ** 2) * s).sum(1), 2000, until=R.CONDITIONCOV) & R.CONDITIONCOV


@pytest.mark.parametrize("case", ["nan", "inf", "mixed"])
def test_history_with_nan_and_inf_fitness(case):
    r = np.random.default_rng(3)

    def f(X):
        v = O.sphere(X - 0.4)
        k = r.integers(0, len(v), 2)
        if case == "nan":
            v[k[0]] = np.nan
        elif case == "inf":
            v[k] = (np.inf, -np.inf)
        else:
            v[k] = (np.nan, np.inf) if r.random() < 0.5 else (-np.inf, np.nan)
        return v
    _drive(5, 9, f, 30)


def test_every_bit_fired_somewhere_in_this_module():
    assert SEEN == set(R.BITS), f"never fired: {sorted(set(R.BITS) - SEEN)}"


# ------------------------------------------------------------------------------------------------ restart in place
_STATE_KEYS = ("mean", "sigma", "C", "p_sigma", "pc", "B", "d", "generation")


@pytest.mark.parametrize("D,lam,lam2", [(10, 10, 20), (10, 20, 6), (128, 4096, 8192)])
def test_restart_equals_a_fresh_instance(D, lam, lam2):
    es = _es(D, lam, seed=3)
    for _ in range(5):
        es.tell(O.sphere(es.ask().cpu().numpy() - 0.3))
    m2 = np.random.default_rng(1).uniform(0, 1, D)
    es.restart(lam2, m2, 0.05)
    fresh = _es(D, lam2, seed=3, mean=m2, sigma=0.05)
    a, b = es.state(), fresh.state()
    for k in _STATE_KEYS:
        assert np.array_equal(a[k], b[k]), k
    fa, fb = es.stop_flags(), fresh.stop_flags()
    assert fa[0] == fb[0] == 0 and fa[2] == fb[2] and np.array_equal(fa[1], fb[1])
    assert es.popsize == lam2 and es.ask().shape == (lam2, D)
    z = torch.tensor(np.random.default_rng(2).standard_normal((lam2, D)), device="cuda")
    Xa, Xb = es.ask(z).cpu().numpy(), fresh.ask(z).cpu().numpy()
    assert np.array_equal(Xa, Xb)
    f = O.sphere(Xa - 0.3)
    es.tell(f)
    fresh.tell(f)
    a, b = es.state(with_Y=True), fresh.state(with_Y=True)
    for k in _STATE_KEYS + ("Y",):
        assert np.array_equal(a[k], b[k]), k
    assert es.stop_flags()[0] == fresh.stop_flags()[0]
    es.close()
    fresh.close()


def test_restart_never_repeats_a_draw():
    D, lam, seed = 6, 8, 11
    es = _es(D, lam, seed)
    for _ in range(4):
        es.tell(O.sphere(es.ask().cpu().numpy()))
    es.restart(12, np.zeros(D), 1.0)                       # B = I, d = 1, m = 0, σ = 1: x = z exactly
    X = es.ask().cpu().numpy()
    np.testing.assert_allclose(X.ravel(), _philox_normals(D * 12, seed, 4), rtol=0, atol=1e-13)   # the draw counter went on
    earlier = np.concatenate([_philox_normals(D * lam, seed, g).reshape(lam, D) for g in range(4)] +
                             [_philox_normals(D * 12, seed, 0).reshape(12, D)])
    for row in X:
        assert not (np.abs(earlier - row).max(1) < 1e-9).any()
    es.close()


# ------------------------------------------------------------------------------------------------ no restart: parent arithmetic
# SHA-256 over X of generation 201 and the state after 200 tells (mean, σ, C, p_σ, p_c, B, d, Y), built-in draws, host
# Rastrigin from mean 3, σ 2, seed 7; computed with the parent commit's libkbo.so on an H100 by
# `tools/cma_restart_cost.py --digest`, whose `digest` this test calls.
PARENT_DIGESTS = {
    (128, 4096): "52869268757fdb4109777c209b92b556b5c227e24ce354398db6885544a62ae3",
    (10, 10): "1e666cfcae624a194f1fef1d3de8434cee9a0cf3e8ebb13b7e5c8e087f082185",
}


def _cost_tool():
    spec = importlib.util.spec_from_file_location("cma_restart_cost", os.path.join(ROOT, "tools", "cma_restart_cost.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("D,lam", list(PARENT_DIGESTS))
def test_no_restart_is_bit_identical_to_the_parent(D, lam):
    es = _es(D, lam, seed=7, mean=3.0, sigma=2.0)
    got = _cost_tool().digest(es)
    es.close()
    assert got == PARENT_DIGESTS[(D, lam)]


# ------------------------------------------------------------------------------------------------ parity across restarts
def _rotated_rastrigin(D, seed=5):
    r = np.random.default_rng(seed)
    Q = np.linalg.qr(r.standard_normal((D, D)))[0]
    xs = r.uniform(0.3, 0.7, D)
    return lambda X: O.rastrigin(((X - xs) @ Q.T) * 10.24)


@pytest.mark.parametrize("strategy,restarts", [("ipop", 3), ("bipop", 4)])
def test_restarts_pass_resynchronised_parity(strategy, restarts):
    D = 10
    f = _rotated_rastrigin(D)
    sched = R.Schedule(strategy, D, sigma0=1.0 / 6.0, random_state=1)
    es = _es(D, sched.lam0, seed=1)
    ck = Checker(es, 1.0 / 6.0)
    r = np.random.default_rng(2)
    runs, g_run, prev = [], 0, None
    while len(runs) < restarts:
        lam = es.popsize
        z = r.standard_normal((lam, D))
        X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
        st = es.state(with_Y=True)
        ev = np.linalg.eigvalsh(st["C"])
        if prev is not None:
            ref, alt, cond = prev
            err = _errors(ref, st, cond)
            if alt is not None:
                err2 = _errors(alt, st, cond)
                if max(err2[k] / LIMITS[k] for k in LIMITS) < max(err[k] / LIMITS[k] for k in LIMITS):
                    err = err2
            for k in LIMITS:
                assert err[k] <= LIMITS[k], f"{strategy} run {len(runs)} generation {st['generation']}: {k} {err[k]:.3g}"
        fx = f(X)
        es.tell(fx)
        g_run += 1
        cond = ev[-1] / ev[0]
        zn2 = (z * z).sum(1)
        ref = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2)
        p = ref.p
        h_left = np.linalg.norm(ref.p_sigma) / np.sqrt(1 - (1 - p.c_sigma) ** (2 * (st["generation"] + 1)))
        thr = (1.4 + 2 / (D + 1)) * p.chi_n
        alt = None
        if abs(h_left - thr) <= TOL_PS * EPS * cond * h_left:
            alt = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2, h_sigma=0.0 if h_left < thr else 1.0)
        prev = (ref, alt, cond)
        if ck.after_tell(fx):
            lam2, m2, s2 = sched.next_run(lam, g_run)
            es.restart(lam2, m2, s2)
            ck.start(s2)
            runs.append((g_run, lam2, s2))
            g_run, prev = 0, None
            st = es.state()
            assert st["generation"] == 0 and np.array_equal(st["mean"], m2) and st["sigma"] == s2
        assert g_run < 3000, f"{strategy}: run {len(runs)} did not stop"
    es.close()
    replay = R.Schedule(strategy, D, sigma0=1.0 / 6.0, random_state=1)
    lam = replay.lam0
    for g, lam2, s2 in runs:
        want = replay.next_run(lam, g)
        assert (want[0], want[2]) == (lam2, s2)
        lam = lam2


# ------------------------------------------------------------------------------------------------ gRPC
def _experiment(name, D, settings):
    from kubeflow_b200.suggestion import api_pb as api
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "cmaes"
    for k, v in settings.items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for i in range(D):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = f"x{i}", api.DOUBLE
        p.feasible_space.min, p.feasible_space.max = "0", "1"
    return e


@pytest.fixture(scope="module")
def service():
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    svc = CmaesService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield svc, SuggestionStub(ch)
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("strategy,D,popsize,objective", [("ipop", 2, None, "round"), ("bipop", 2, None, "round"),
                                                          ("ipop", 32, None, "constant"), ("bipop", 32, None, "constant"),
                                                          ("ipop", 2, 4096, "constant")])
def test_grpc_experiment_restarts_on_the_schedule(service, monkeypatch, strategy, D, popsize, objective):
    from kubeflow_b200 import cmaes as cm
    from kubeflow_b200.suggestion import api_pb as api
    svc, stub = service
    restarts = []
    orig = cm.CmaEs.restart

    def spy(self, lam, mean, sigma):
        flags = self.stop_flags()[0]
        restarts.append((flags, self.popsize, lam, np.array(mean), sigma))
        return orig(self, lam, mean, sigma)
    monkeypatch.setattr(cm.CmaEs, "restart", spy)
    settings = {"restart_strategy": strategy, "random_state": 5, **({"popsize": popsize} if popsize else {})}
    name = f"grpc-{strategy}-{D}-{popsize}"
    exp = _experiment(name, D, settings)
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    xs = np.linspace(0.2, 0.8, D)
    fobj = (lambda U: np.round(((U - xs) ** 2).sum(1), 3)) if objective == "round" else (lambda U: np.full(len(U), 1.5))
    k, run_gens, gens = 0, [], 0
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=0)
    stub.GetSuggestions(req)
    while len(restarts) < 3:
        st = svc._exps[name]
        n_before = len(restarts)
        req = api.GetSuggestionsRequest(experiment=exp, current_request_number=len(st.queue))
        rep = stub.GetSuggestions(req)
        U = np.array([[float(a.value) for a in pa.assignments] for pa in rep.parameter_assignments])
        req = api.GetSuggestionsRequest(experiment=exp, current_request_number=0)   # only the new trials: names are remembered
        for pa, v in zip(rep.parameter_assignments, fobj(U)):
            t = req.trials.add()
            t.name = f"t{k}"
            k += 1
            t.spec.objective.objective_metric_name = "loss"
            t.spec.parameter_assignments.assignments.extend(pa.assignments)
            t.status.condition = api.SUCCEEDED
            m = t.status.observation.metrics.add()
            m.name, m.value = "loss", repr(float(v))
        stub.GetSuggestions(req)
        gens += 1
        if len(restarts) > n_before:
            run_gens.append(gens)
            gens = 0
        assert sum(run_gens) + gens < 1500, "no restart"
    sched = R.Schedule(strategy, D, popsize, 1.0 / 6.0, 5)
    lam = sched.lam0
    for (flags, lam_run, lam2, mean, sigma), g in zip(restarts, run_gens):
        assert flags != 0 and lam_run == lam
        want = sched.next_run(lam, g)
        assert (want[0], want[2]) == (lam2, sigma) and np.array_equal(want[1], mean)
        lam = lam2
    if popsize == 4096:
        assert [r[2] for r in restarts] == [8192, 8192, 8192]
    assert svc._exps[name].es.popsize == lam
