"""GPU: kbo_lml_grad_batch (GPEngine.lml_grad_batch) and ``Optimizer(theta_fit="skopt")``.

* The batch against one kbo_fit + kbo_lml_grad per θ and against ``oracle.gp_oracle.lml_and_grad``, at the bounds of
  tests/test_gpu_fit_scale.py: LML to 1e-9 relative, gradient to 1e-11 of max|g|.
* Each θ's (LML, gradient) bit-identical alone, at every position of a batch of 8, and run to run; a non-positive-definite θ
  mid-batch gives −inf, a zero gradient and its pivot without touching its neighbours; an over-budget batch fails cleanly.
* The skopt fit on the sklearn golden cases (tests/golden/thetafit_cases.npz) and at the workload of record, and over gRPC.
"""
import grpc
import numpy as np
import pytest

from kubeflow_b200 import thetafit as TF
from kubeflow_b200 import workload
from kubeflow_b200._lib import KboError
from kubeflow_b200.gp import GPEngine
from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Real
from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, SkoptService
from oracle import gp_oracle as O
from tests import _thetafit_ref as R
from tests.test_grpc_service import add_trial, make_experiment
from tests.test_thetafit_oracle import CASES, FLAT, TOL_NEG_LML, TOL_THETA

pytestmark = pytest.mark.gpu

TOL_LML = 1e-9
TOL_GRAD = 1e-11


@pytest.fixture(scope="module")
def eng():
    e = GPEngine(0, scratch_limit=16 << 30)
    yield e
    e.close()


def _history(N, D, seed):
    r = np.random.default_rng(seed)
    X = r.random((N, D))
    y = np.sin(3 * X.sum(1) / np.sqrt(D)) + 0.1 * r.standard_normal(N)
    return X, y


def _thetas(G, D, ard, seed):
    """θ in the regime test_gpu_fit_scale.py's bounds were measured in (noise >= 1e-3): lower noise on a dense history makes K
    ill-conditioned enough that two correct FP64 computations of the gradient differ by more than 1e-11 of max|g|."""
    r = np.random.default_rng(seed + 1)
    out = []
    for _ in range(G):
        ls = 0.3 * np.sqrt(D) * (r.uniform(0.5, 2.0, D) if ard else r.uniform(0.5, 2.0))
        out.append(dict(length_scale=np.atleast_1d(ls), amplitude=float(r.uniform(0.5, 3.0)), noise=float(10 ** r.uniform(-3, -1))))
    return out


# (N, D, ard, kernel, G): every N, D, G, both kernels, isotropic and ARD
SHAPES = [(1, 1, False, "matern52", 1), (63, 17, True, "rbf", 3), (64, 32, False, "matern52", 8), (65, 1, True, "matern52", 3),
          (1000, 17, True, "matern52", 3), (1000, 32, False, "rbf", 8), (4097, 17, True, "rbf", 3), (8192, 32, True, "matern52", 3),
          (8192, 17, False, "rbf", 1)]


@pytest.mark.parametrize("N,D,ard,kind,G", SHAPES)
def test_batch_against_fit_and_oracle(eng, N, D, ard, kind, G):
    X, y = _history(N, D, N + D)
    ths = _thetas(G, D, ard, N)
    eng.kernel = kind
    lml, grad = eng.lml_grad_batch(X, y, ths)
    assert lml.shape == (G,) and grad.shape == (G, 2 + (D if ard else 1))
    ref = GPEngine(0, kernel=kind)
    try:
        for g, th in enumerate(ths):
            ref.length_scale, ref.amplitude, ref.noise = th["length_scale"], th["amplitude"], th["noise"]
            ref.tell(X, y)
            l1, g1 = ref.lml_grad()
            assert abs(lml[g] - l1) <= TOL_LML * max(1.0, abs(l1)), (g, lml[g], l1)
            assert np.abs(grad[g] - g1).max() <= TOL_GRAD * np.abs(g1).max(), (g, np.abs(grad[g] - g1).max())
            if N <= 4097 and g == 0:
                lo, go = O.lml_and_grad(X, y, kind=kind, length_scale=th["length_scale"] if ard else th["length_scale"][0],
                                        amplitude=th["amplitude"], noise=th["noise"], chunk=256)
                assert abs(lml[g] - lo) <= TOL_LML * max(1.0, abs(lo))
                assert np.abs(grad[g] - go).max() <= TOL_GRAD * np.abs(go).max()
    finally:
        ref.close()


@pytest.mark.parametrize("N,D,kind", [(1000, 17, "matern52"), (2049, 32, "rbf")])
def test_each_theta_is_bit_identical_in_any_batch(eng, N, D, kind):
    X, y = _history(N, D, 5)
    ths = _thetas(8, D, True, 9)
    eng.kernel = kind
    lml8, grad8, info8 = eng.lml_grad_batch(X, y, ths, return_info=True)
    assert not info8.any()
    again = eng.lml_grad_batch(X, y, ths)
    rev = eng.lml_grad_batch(X, y, ths[::-1])
    for g, th in enumerate(ths):
        l1, g1 = eng.lml_grad_batch(X, y, [th])
        assert l1[0] == lml8[g] and np.array_equal(g1[0], grad8[g]), g
        assert again[0][g] == lml8[g] and np.array_equal(again[1][g], grad8[g])
        assert rev[0][7 - g] == lml8[g] and np.array_equal(rev[1][7 - g], grad8[g])


def test_non_pd_theta_mid_batch(eng):
    p = 70
    X, y = O.not_pd_at(100, p)
    eng.kernel = "rbf"
    good = [dict(length_scale=np.ones(1), amplitude=1.0, noise=1e-2), dict(length_scale=np.ones(1) * 0.7, amplitude=2.0, noise=1e-3)]
    bad = dict(length_scale=np.ones(1), amplitude=1.0, noise=0.0)
    lml, grad, info = eng.lml_grad_batch(X, y, [good[0], bad, good[1]], return_info=True)
    assert lml[1] == -np.inf and not grad[1].any() and info[1] == p
    assert info[0] == info[2] == 0
    l2, g2 = eng.lml_grad_batch(X, y, good)
    assert lml[0] == l2[0] and lml[2] == l2[1] and np.array_equal(grad[[0, 2]], g2)


def test_over_budget_batch_fails_cleanly():
    X, y = _history(4096, 8, 1)
    ths = _thetas(3, 8, True, 2)
    e = GPEngine(0, scratch_limit=64 << 20)       # one θ at N = 4096 takes about 384 MiB
    try:
        with pytest.raises(KboError, match="need [0-9]+ bytes"):
            e.lml_grad_batch(X, y, ths)
        Xs, ys = X[:512], y[:512]
        l, g = e.lml_grad_batch(Xs, ys, ths)                        # the handle stays usable
        e.length_scale, e.amplitude, e.noise = ths[1]["length_scale"], ths[1]["amplitude"], ths[1]["noise"]
        e.tell(Xs, ys)
        l1, g1 = e.lml_grad()
        assert abs(l[1] - l1) <= TOL_LML * abs(l1)
    finally:
        e.close()


@pytest.mark.parametrize("name", sorted(CASES))
def test_skopt_fit_on_the_golden_cases(eng, name):
    c = CASES[name]
    eng.kernel = "matern52"
    res = TF.fit(TF.engine_batch_fn(eng, c["X"], c["y"]), c["X"].shape[1], int(c["seed"]), 2)
    for i, s in enumerate(res.starts):
        np.testing.assert_array_equal(s.theta0, c["theta0"][i])
        assert abs(s.fun - c["neg_lml"][i]) <= TOL_NEG_LML * abs(c["neg_lml"][i]), (i, s.fun, c["neg_lml"][i])
        assert np.abs(s.theta - c["theta"][i]).max() <= FLAT.get((name, i), TOL_THETA)
    assert abs(res.lml - c["lml"]) <= TOL_NEG_LML * abs(c["lml"])
    assert np.abs(res.theta - c["kernel_theta"]).max() <= 1e-3     # a flat valley at worst (tests/test_thetafit_oracle.py)
    # the Optimizer drives the same fit: tell the golden history on Real(0, 1) dimensions (the identity transform) and ask
    opt = Optimizer([Real(0.0, 1.0)] * c["X"].shape[1], n_initial_points=1, acq_func="EI", random_state=int(c["random_state"]),
                    theta_fit="skopt", n_points=1024)
    opt.tell(c["X"].tolist(), c["y"].tolist())
    assert np.array_equal(opt._Xt, c["X"])
    opt.ask()
    lt = opt.last_theta
    assert lt["winner"] == res.winner and lt["lml"] == res.lml and lt["batch_calls"] == res.batch_calls
    assert lt["amplitude"] == np.exp(res.theta[0]) and np.array_equal(lt["length_scale"], np.exp(res.theta[1:-1]))
    opt._engine.close()


@pytest.mark.parametrize("N", [2048, 8192])
def test_skopt_fit_at_the_workload_of_record(eng, N):
    D = 32
    X, y = workload.trials(N, D)
    eng.kernel = "matern52"
    seed = TF.estimator_seed(0)
    lock = TF.fit(TF.engine_batch_fn(eng, X, y), D, seed, 2)
    b = TF.bounds(D)
    # the reported LML is the FP64 LML at the returned θ
    f, g = R.objective(X, y, lock.theta) if N <= 2048 else TF.to_objective(*[v[0] for v in eng.lml_grad_batch(X, y, [TF.theta_dict(lock.theta)])],
                                                                         float(np.exp(lock.theta[-1])))
    assert abs(-f - lock.lml) <= TOL_LML * abs(lock.lml)
    # projected gradient (of −LML) near zero: interior coordinates small, active bounds pushed outward
    at_lo, at_hi = lock.theta <= b[:, 0] + 1e-8, lock.theta >= b[:, 1] - 1e-8
    interior = ~(at_lo | at_hi)
    scale = max(1.0, abs(lock.lml))
    assert np.abs(g[interior]).max(initial=0.0) <= 1e-3 * scale, g[interior]
    assert (g[at_lo] >= -1e-3 * scale).all() and (g[at_hi] <= 1e-3 * scale).all()
    for s in lock.starts:
        f0 = TF.engine_batch_fn(eng, X, y)([s.theta0])[0][0]
        assert s.fun <= f0
    seq = TF.fit(TF.engine_batch_fn(eng, X, y), D, seed, 2, lockstep=False)
    assert lock.winner == seq.winner and np.array_equal(lock.theta, seq.theta) and lock.lml == seq.lml
    for a, s in zip(lock.starts, seq.starts):
        assert np.array_equal(a.theta, s.theta) and (a.fun, a.nit, a.nfev, a.status) == (s.fun, s.nit, s.nfev, s.status)
    assert lock.batch_calls == max(s.nfev for s in lock.starts) < seq.batch_calls


def test_skopt_theta_fit_over_grpc():
    sk = SkoptService()
    server, port = serve(DispatchService([sk]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    stub = SuggestionStub(ch)
    settings = {"n_initial_points": 6, "acq_func": "EI", "random_state": 4, "n_points": 4096, "theta_fit": "skopt",
                "candidate_backend": "numpy"}
    exp = make_experiment("bayesianoptimization", settings, name="bo-skopt-theta")
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=2)
    names = [f"x{i}" for i in range(4)]
    from kubeflow_b200.space import Space
    direct = Optimizer(Space([Real(0.01, 0.1), Real(-1.0, 1.0), Real(10.0, 20.0), Real(0.0, 5.0)]), n_initial_points=6, acq_func="EI",
                       random_state=4, n_points=4096, theta_fit="skopt", candidate_backend="numpy")
    n = 0
    try:
        for step in range(6):
            reply = stub.GetSuggestions(req)
            got = [[float(a.value) for a in pa.assignments] for pa in reply.parameter_assignments]
            want = direct.ask(n_points=2)                 # the Optimizer driven directly with the same trials
            assert np.allclose(got, np.asarray(want, dtype=np.float64), rtol=1e-12, atol=0), step
            opt = sk._services["bo-skopt-theta"].skopt_optimizer
            if step >= 3:            # model-based: θ refitted once per new told history, the lie appended at that θ
                assert opt.theta_refits == direct.theta_refits == step - 2 and opt.last_fit == "append"
                assert opt.last_theta["lml"] == direct.last_theta["lml"] and len(opt.last_theta["starts"]) == 3
            rows = []
            for row in got:
                vals = dict(zip(names, row))
                n += 1
                loss = float(np.sin(vals["x1"] * 3) + vals["x3"] / 5)
                add_trial(req, f"t{n}", vals, loss)
                rows.append((row, loss))
            direct.tell([r for r, _ in rows], [v for _, v in rows])
        refits = opt.theta_refits
        req2 = api.GetSuggestionsRequest(experiment=exp, current_request_number=1)
        req2.trials.extend(req.trials)
        stub.GetSuggestions(req2)                       # no new trials: θ reused
        assert opt.theta_refits == refits + 1
        stub.GetSuggestions(req2)
        assert opt.theta_refits == refits + 1
    finally:
        ch.close()
        server.stop(0)
        direct._engine and direct._engine.close()
