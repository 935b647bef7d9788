"""CPU: skopt's θ fit (``theta_fit="skopt"``) off the device.

* The plain restatement in ``tests/_thetafit_ref.py`` (FP64 NumPy LML and gradient, SciPy L-BFGS-B, one start after another)
  against the REAL scikit-learn 1.9 GaussianProcessRegressor configured as skopt's default GP (tests/golden/thetafit_cases.npz,
  made by tools/make_golden_thetafit.py): the starts exactly, each start's −LML to 1e-9 relative, each start's final θ to 1e-6
  where its optimum is well defined, and the winner.
* ``kubeflow_b200.thetafit``'s lockstep driver against the same starts run one after another, on a NumPy stand-in for the
  engine with random delays in every thread: bit for bit.
* Validation over a real in-process gRPC server.

Where trajectories separate.  In the near-noiseless cases the fitted noise sits on its lower bound (1e-5) and the LML is flat
along some length scales near the optimum: L-BFGS-B stops there on its relative-reduction test (factr·eps ≈ 2.2e-9 of |f|),
and where inside the flat valley it stops depends on the last bits of each gradient.  The NumPy and sklearn evaluations differ
in those bits (summation order), so final θ there agree only to ~1e-4 (3.4e-5 the worst seen with the NumPy restatement,
1.7e-4 with the device's LML on an H100) while −LML agrees to 5e-10.  Those start runs are listed in FLAT with the bound
they are held to; the test also shows the valley is flat, by evaluating the
restatement at sklearn's θ and finding sklearn's −LML.  Likewise, when two starts of a case converge to the same optimum their
−LML differ in the last bits and np.argmin may pick either; the winner is then held to the same θ and −LML instead of the same
index.

Non-positive-definite θ.  No θ inside skopt's bounds is: the noise (>= 1e-5) bounds the Gram matrix's smallest eigenvalue from
below by far more than the Cholesky's rounding (~N·amp·eps <= 3.4e-11 at N = 150, amp = 1000).  The (+inf, 0) path is covered
by the stand-in below, which reports such θ on purpose, and on the device by tests/test_gpu_thetafit.py.
"""
import os
import random
import time

import grpc
import numpy as np
import pytest

from kubeflow_b200 import thetafit as TF
from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Real
from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, SkoptService
from tests import _thetafit_ref as R
from tests.test_grpc_service import make_experiment

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "thetafit_cases.npz")
CASES = R.golden_cases(GOLDEN)
TOL_THETA = 1e-6
TOL_NEG_LML = 1e-9
# (case, start) -> θ bound for the near-noiseless runs that stop in a flat valley (see the module docstring)
FLAT = {("smooth_n20_d1", 0): 1e-3, ("smooth_n20_d1", 2): 1e-3, ("smooth_n150_d6", 2): 1e-3, ("smooth_n20_d3", 1): 1e-3}


@pytest.fixture(scope="module")
def oracle_fits():
    return {name: R.skopt_theta_fit(c["X"], c["y"], seed=int(c["seed"])) for name, c in CASES.items()}


def test_golden_cases_cover_the_shapes():
    shapes = {c["X"].shape for c in CASES.values()}
    assert {(20, 1), (60, 3), (150, 6)} <= shapes
    assert any(np.isclose(c["kernel_theta"][-2], np.log(100.0)) for c in CASES.values()), "an irrelevant dimension's ℓ reaches 100"
    assert any(c["kernel_theta"][-1] > np.log(1e-2) for c in CASES.values()), "a noisy target"


@pytest.mark.parametrize("name", sorted(CASES))
def test_starts_are_sklearns(name):
    c = CASES[name]
    D = c["X"].shape[1]
    assert int(c["seed"]) == TF.estimator_seed(int(c["random_state"]))
    np.testing.assert_array_equal(TF.starts(D, int(c["seed"]), 2), c["theta0"])
    np.testing.assert_array_equal(TF.bounds(D), R.log_bounds(D))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_against_sklearn(name, oracle_fits):
    c, r = CASES[name], oracle_fits[name]
    for i, s in enumerate(r["starts"]):
        np.testing.assert_array_equal(s["theta0"], c["theta0"][i])
        rel = abs(s["neg_lml"] - c["neg_lml"][i]) / abs(c["neg_lml"][i])
        assert rel <= TOL_NEG_LML, f"{name} start {i}: −LML off by {rel:.2e} relative"
        dth = float(np.abs(s["theta"] - c["theta"][i]).max())
        tol = FLAT.get((name, i), TOL_THETA)
        assert dth <= tol, f"{name} start {i}: θ off by {dth:.2e} (> {tol:.0e})"
        if (name, i) in FLAT:       # the valley is flat: the restatement at sklearn's θ gives sklearn's −LML
            f, _ = R.objective(c["X"], c["y"], c["theta"][i])
            assert abs(f - c["neg_lml"][i]) <= TOL_NEG_LML * abs(c["neg_lml"][i])
    w_ref = int(np.argmin(c["neg_lml"]))
    if r["winner"] != w_ref:        # two starts reached the same optimum: np.argmin may take either
        assert abs(c["neg_lml"][r["winner"]] - c["neg_lml"][w_ref]) <= TOL_NEG_LML * abs(c["neg_lml"][w_ref])
        assert np.abs(c["theta"][r["winner"]] - c["theta"][w_ref]).max() <= 1e-3
    assert abs(r["lml"] - c["lml"]) <= TOL_NEG_LML * abs(c["lml"])
    assert np.abs(r["theta"] - c["kernel_theta"]).max() <= 1e-3


def _stand_in(X, y, delays, calls):
    """NumPy stand-in for GPEngine.lml_grad_batch: each θ evaluated alone by the restatement, after a random delay; θ with
    amplitude above e^5 report "not positive definite" (+inf, 0) as the device would."""
    def batch_fn(thetas):
        calls.append(len(thetas))
        out = []
        for t in thetas:
            if delays:
                time.sleep(random.random() * 2e-3)
            out.append((np.inf, np.zeros(len(t))) if t[0] > 5.0 else R.objective(X, y, t))
        return out
    return batch_fn


@pytest.mark.parametrize("name,restarts,maxiter", [("noisy_n60_d3", 2, None), ("smooth_n20_d1", 4, None), ("smooth_n20_d3", 2, 7),
                                                   ("irrelevant_n60_d3", 0, None)])
def test_lockstep_equals_sequential(name, restarts, maxiter):
    c = CASES[name]
    seed, D = int(c["seed"]), c["X"].shape[1]
    seq_calls, lock_calls = [], []
    seq = TF.fit(_stand_in(c["X"], c["y"], False, seq_calls), D, seed, restarts, maxiter, lockstep=False)
    random.seed(1)
    lock = TF.fit(_stand_in(c["X"], c["y"], True, lock_calls), D, seed, restarts, maxiter, lockstep=True)
    assert lock.winner == seq.winner and np.array_equal(lock.theta, seq.theta) and lock.lml == seq.lml
    for a, b in zip(lock.starts, seq.starts):
        assert np.array_equal(a.theta0, b.theta0) and np.array_equal(a.theta, b.theta)
        assert (a.fun, a.nit, a.nfev, a.status) == (b.fun, b.nit, b.nfev, b.status)
        if maxiter is not None:
            assert a.nit <= maxiter
    assert set(seq_calls) == {1} and seq.batch_calls == sum(s.nfev for s in seq.starts)
    # one round per evaluation of the longest start; every round carries every start still running
    assert lock.batch_calls == len(lock_calls) == max(s.nfev for s in lock.starts)
    assert sum(lock_calls) == sum(s.nfev for s in lock.starts)
    assert lock_calls[0] == restarts + 1


def test_lockstep_passes_a_batch_failure_to_every_start():
    def bad(thetas):
        raise RuntimeError("device failure")
    with pytest.raises(RuntimeError, match="device failure"):
        TF.fit(bad, 2, 5, 2)


def test_objective_conversion():
    lml, g = 3.0, np.array([1.0, 2.0, 3.0, 4.0])          # device order: amp, noise, ℓ1, ℓ2
    f, gs = TF.to_objective(lml, g, 1e-10)
    assert f == -3.0 and np.array_equal(gs, -np.array([1.0, 3.0, 4.0, 2.0 * 0.5]))
    f, gs = TF.to_objective(-np.inf, np.zeros(4), 1.0)
    assert f == np.inf and not gs.any()
    th = TF.theta_dict(np.log([2.0, 0.5, 4.0, 1e-3]))
    assert th["noise"] == 1e-3 + 1e-10 or abs(th["noise"] - (1e-3 + 1e-10)) < 1e-18


def test_optimizer_refuses_combinations_without_a_device():
    dims = [Real(0.0, 1.0), Real(-1.0, 1.0)]
    Optimizer(dims, theta_fit="skopt")
    Optimizer(dims, theta_fit="skopt", theta_restarts=0, theta_fit_maxiter=50)
    for kw, name in ((dict(theta_grid=3), "theta_grid"), (dict(theta_search=2), "theta_search"), (dict(ard=True), "ard"),
                     (dict(length_scale=0.5), "length_scale"), (dict(amplitude=2.0), "amplitude"), (dict(noise=1e-4), "noise")):
        with pytest.raises(ValueError, match=name):
            Optimizer(dims, theta_fit="skopt", **kw)
    for tf in (None, "lbfgs"):
        with pytest.raises(ValueError, match="theta_restarts"):
            Optimizer(dims, theta_fit=tf, theta_restarts=2)
    with pytest.raises(ValueError, match="theta_restarts"):
        Optimizer(dims, theta_fit="skopt", theta_restarts=-1)
    assert Optimizer(dims, theta_fit="lbfgs").theta_fit_maxiter is None     # lbfgs still runs 25 iterations by default
    o = Optimizer(dims, theta_fit="skopt", random_state=3)
    assert o._est_seed == TF.estimator_seed(3) and o.theta_restarts == 2


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([SkoptService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _validate(stub, settings):
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment("bayesianoptimization", settings)))


def _refused(stub, settings, words):
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, settings)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    for w in words:
        assert w in ei.value.details(), ei.value.details()


def test_skopt_theta_fit_is_accepted(stub):
    _validate(stub, {"theta_fit": "skopt"})
    _validate(stub, {"theta_fit": "skopt", "theta_restarts": 0})
    _validate(stub, {"theta_fit": "skopt", "theta_restarts": 5, "theta_fit_maxiter": 100, "kernel": "rbf", "acq_func": "EI"})
    _validate(stub, {"theta_fit": "lbfgs"})


@pytest.mark.parametrize("knob,value", [("theta_grid", 3), ("theta_search", 2), ("ard", 1), ("length_scale", 0.5), ("amplitude", 2.0),
                                        ("noise", 1e-4)])
def test_skopt_theta_fit_refuses_theta_knobs(stub, knob, value):
    _refused(stub, {"theta_fit": "skopt", knob: value}, [knob, "skopt"])


def test_theta_restarts_needs_skopt_theta_fit(stub):
    _refused(stub, {"theta_restarts": 2}, ["theta_restarts"])
    _refused(stub, {"theta_fit": "lbfgs", "theta_restarts": 2}, ["theta_restarts"])
    _refused(stub, {"theta_fit": "skopt", "theta_restarts": -1}, ["theta_restarts"])
    _refused(stub, {"theta_fit": "bfgs"}, ["theta_fit"])


@pytest.mark.parametrize("est", ["RF", "ET"])
def test_tree_estimators_refuse_theta_restarts(stub, est):
    _refused(stub, {"base_estimator": est, "theta_restarts": 2}, ["theta_restarts", est])
    _refused(stub, {"base_estimator": est, "theta_fit": "skopt"}, ["theta_fit", est])
