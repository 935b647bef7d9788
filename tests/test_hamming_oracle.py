"""CPU: ``kernel="hamming"`` (skopt's HammingKernel GP for all-categorical spaces) off the device.

* ``oracle/hamming_oracle.py`` against the REAL scikit-learn 1.9 GaussianProcessRegressor with a restated HammingKernel
  (tests/golden/hamming_cases.npz, made by tools/make_golden_hamming.py): the starts exactly; the LML, its gradient and the
  posterior μ and σ to 1e-12 relative where K is well conditioned; each start's final θ to 1e-6 and −LML to 1e-9.
* The one-hot mapping (``kubeflow_b200.hamming``) against the oracle: the Gram matrix to 1e-15 relative, with one-, two- and
  many-category dimensions, and the gradient per l_j through the RBF gradient of the one-hot columns.
* The sweep-mode choice on both sides of its range, and validation in the Optimizer (without a device) and over gRPC.

Ill-conditioned θ.  At a fitted θ with a large amplitude, small l_j and small noise, K's condition number κ reaches 1e8: two
correct FP64 evaluations of the LML, of the gradient (at the optimum, itself ~1e-5) or of σ then differ by about κ·eps of their
scale, and those values are held to 4·κ·eps instead (κ is computed by the test; 5e5 at one start of c2_d1_n16 puts the LML
there at 1e-11).

Flat valleys.  A dimension the target does not depend on leaves the LML nearly flat in its l_j; there L-BFGS-B stops on its
relative-reduction test at a point that depends on the last bits of each gradient.  The one such start run whose final θ differs
by more than 1e-6 between the oracle and sklearn is listed in FLAT; its −LML still agrees to 1e-9.  When two starts reach the
same optimum np.argmin may pick either: the winner is then held to the same −LML.
"""
import os

import grpc
import numpy as np
import pytest

from kubeflow_b200 import hamming as HM
from kubeflow_b200 import thetafit as TF
from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Categorical, Integer, Real, Space
from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, SkoptService
from oracle import gp_oracle as O
from oracle import hamming_oracle as H

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hamming_cases.npz")
FIELDS = ("categories", "X", "y", "Xc", "random_state", "seed", "theta0", "theta", "neg_lml", "kernel_theta", "lml", "probe_theta",
          "probe_lml", "probe_grad", "mu", "std")
EPS = np.finfo(np.float64).eps
FLAT = {("noisy_d8_n200", 2): 2e-3}   # 1.3e-3 recorded, along l_4 (see tools/make_golden_hamming.py)


def _cases():
    z = np.load(GOLDEN)
    return {str(n): {f: z[f"{n}__{f}"] for f in FIELDS} for n in z["names"]}


CASES = _cases()


def space_of(categories):
    return Space([Categorical([float(v) for v in range(int(c))], name=f"c{j}") for j, c in enumerate(categories)])


def _cond(X, t):
    f = H.fit(X, np.zeros(len(X)) + np.arange(len(X)), t)
    K = f["amp"] * f["Kh"] + (f["noise"] + H.ALPHA) * np.eye(len(X))
    return float(np.linalg.cond(K))


def test_golden_cases_cover_the_shapes():
    cats = {int(c) for case in CASES.values() for c in case["categories"]}
    assert {1, 2, 3, 7} <= cats
    assert {1, 3, 8} <= {case["X"].shape[1] for case in CASES.values()}
    assert max(case["X"].shape[0] for case in CASES.values()) == 512
    # a one-category dimension keeps its start; an irrelevant one reaches the lower bound
    one = CASES["one_d3_n80"]
    np.testing.assert_array_equal(one["theta"][:, 1], one["theta0"][:, 1])
    assert np.isclose(CASES["mixed_d8_n512"]["kernel_theta"][6], np.log(1e-5))


@pytest.mark.parametrize("name", sorted(CASES))
def test_starts_are_sklearns(name):
    c = CASES[name]
    D = c["X"].shape[1]
    assert int(c["seed"]) == TF.estimator_seed(int(c["random_state"]))
    np.testing.assert_array_equal(TF.starts(D, int(c["seed"]), 2, HM.LS_BOUNDS), c["theta0"])
    np.testing.assert_array_equal(H.starts(D, int(c["seed"])), c["theta0"])
    np.testing.assert_array_equal(TF.bounds(D, HM.LS_BOUNDS), H.log_bounds(D))


@pytest.mark.parametrize("name", sorted(CASES))
def test_lml_gradient_and_posterior(name):
    c = CASES[name]
    for t, lml, g in zip(c["probe_theta"], c["probe_lml"], c["probe_grad"]):
        lo, go = H.lml_and_grad(c["X"], c["y"], t)
        rel = max(1e-12, 4 * _cond(c["X"], t) * EPS)
        assert abs(lo - lml) <= rel * abs(lml), (t, lo, lml)
        tol = rel * max(1.0, float(np.abs(g).max()))
        assert np.abs(go - g).max() <= tol, (t, np.abs(go - g).max(), tol)
    f = H.fit(c["X"], c["y"], c["kernel_theta"])
    mu, sd = H.predict(f, c["Xc"])
    rel = max(1e-12, 4 * _cond(c["X"], c["kernel_theta"]) * EPS)
    assert np.abs(mu - c["mu"]).max() <= rel * np.abs(c["mu"]).max()
    assert np.abs(sd - c["std"]).max() <= rel * np.abs(c["std"]).max()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_fit_against_sklearn(name):
    c = CASES[name]
    r = H.skopt_fit(c["X"], c["y"], seed=int(c["seed"]))
    for i, s in enumerate(r["starts"]):
        np.testing.assert_array_equal(s["theta0"], c["theta0"][i])
        assert abs(s["neg_lml"] - c["neg_lml"][i]) <= 1e-9 * abs(c["neg_lml"][i])
        dth = float(np.abs(s["theta"] - c["theta"][i]).max())
        assert dth <= FLAT.get((name, i), 1e-6), (name, i, dth)
    w_ref = int(np.argmin(c["neg_lml"]))
    if r["winner"] != w_ref:
        assert abs(c["neg_lml"][r["winner"]] - c["neg_lml"][w_ref]) <= 1e-9 * abs(c["neg_lml"][w_ref])
    assert abs(r["lml"] - c["lml"]) <= 1e-9 * abs(c["lml"])


# ---- the one-hot mapping ---------------------------------------------------------------------------------------------------
MAP_CATS = [1, 2, 3, 7, 2, 1, 5, 3]


def _codes(r, n, cats):
    return np.stack([r.integers(0, c, n) for c in cats], axis=1).astype(np.float64)


def test_one_hot_gram_equals_the_hamming_gram():
    """exp of the mapped RBF exponent against exp(−Σ l_j·[x_j ≠ y_j]).  The mapped exponent carries a few ulp of relative error
    per term, so the kernel values agree to S·few eps; S ≤ 1 here (weights up to 0.2) gives the 1e-15 bound, and the second
    half checks the whole weight range in the exponent itself, to 8 eps relative."""
    r = np.random.default_rng(0)
    sp = space_of(MAP_CATS)
    hm = HM.HammingMap(sp)
    A, B = _codes(r, 60, MAP_CATS), _codes(r, 50, MAP_CATS)
    A[:5] = B[:5]                                                   # exact matches
    for l in (r.uniform(0.0, 0.2, len(MAP_CATS)), 0.1):
        Kh = H.kernel(A, B, l, amp=2.0)
        Km = O.kernel_matrix(sp.transform(A.tolist()), sp.transform(B.tolist()), hm.length_scale(l), kind="rbf", amplitude=2.0)
        assert np.abs(Km - Kh).max() <= 1e-15 * np.abs(Kh).max() and (np.abs(Km - Kh) <= 1e-15 * Kh).all()
    for l in (np.exp(r.uniform(np.log(1e-5), np.log(1e5), len(MAP_CATS))), 1e-5, 1e5):
        S = H.mismatch_sum(A, B, l)
        ls = hm.length_scale(l)
        At, Bt = sp.transform(A.tolist()) / ls, sp.transform(B.tolist()) / ls
        Sm = 0.5 * ((At[:, None, :] - Bt[None, :, :]) ** 2).sum(-1)
        assert (np.abs(Sm - S) <= 8 * EPS * S).all()


def test_gradient_through_the_one_hot_columns():
    """The per-column RBF gradient of the one-hot GP, mapped to l_j (HammingMap.grad) and converted to sklearn's order
    (thetafit.to_objective), is the oracle's Hamming gradient; a one-category dimension's is exactly zero."""
    r = np.random.default_rng(1)
    sp = space_of(MAP_CATS)
    hm = HM.HammingMap(sp)
    X = _codes(r, 120, MAP_CATS)
    y = np.sin(X @ np.linspace(0.3, 1.0, len(MAP_CATS))) + 0.1 * r.standard_normal(120)
    for t in (np.log([1.5] + [1.0] * len(MAP_CATS) + [0.01]), np.r_[0.3, r.uniform(-3, 2, len(MAP_CATS)), -4.0]):
        th = TF.theta_dict(t)
        lml, g = O.lml_and_grad(sp.transform(X.tolist()), y, kind="rbf", length_scale=hm.length_scale(th["length_scale"]),
                                amplitude=th["amplitude"], noise=th["noise"])
        f, gs = TF.to_objective(lml, np.concatenate([g[:2], hm.grad(g[2:])]), float(np.exp(t[-1])))
        lh, gh = H.lml_and_grad(X, y, t)
        assert abs(-f - lh) <= 1e-11 * abs(lh)
        assert np.abs(-gs - gh).max() <= 1e-10 * np.abs(gh).max()
        assert gs[1 + 0] == 0.0 and gs[1 + 5] == 0.0              # the one-category dimensions


def test_sweep_mode_on_both_sides_of_the_range():
    hm = HM.HammingMap(space_of([1, 2, 3, 7]))                      # three dimensions can differ
    lo, hi = HM.TC_RANGE
    for l, mode in ((lo / 3 * 0.999, "f64"), (lo / 3 * 1.001, "auto"), (1.0, "auto"), (hi / 3 * 0.999, "auto"), (hi / 3 * 1.001, "f64"),
                    (1e-5, "f64"), (1e5, "f64"), ([1e5, 0.1, 0.1, 0.1], "auto")):   # the c = 1 weight does not count
        assert hm.var_mode(l, "auto") == mode, (l, mode)
        assert hm.var_mode(l, "tc") == "tc" and hm.var_mode(l, "f64") == "f64"
    np.testing.assert_allclose(hm.length_scale([4.0, 2.0, 4.0, 0.25]), [1.0, 0.5, 0.5, 0.5, 0.5, 2, 2, 2, 2, 2, 2, 2], rtol=1e-15)


@pytest.mark.parametrize("l1", [1.0, 1e5, 1e-5])
def test_one_category_columns_drop_out(l1):
    """A one-category dimension's column: the sampled candidates are encoded as the told rows are (to_unit gives 1, the sampler
    the index 0), its length scale stays 1 whatever its weight, and its weight has a zero gradient — so on candidates drawn
    the way the Optimizer draws them, the one-hot Gram equals the Hamming Gram at any weight of that dimension."""
    r = np.random.default_rng(2)
    sp = space_of(MAP_CATS)
    hm = HM.HammingMap(sp)
    U = hm.candidates(sp.rvs_transformed(400, r, np.float64))
    np.testing.assert_array_equal(sp.transform(sp.inverse_transform(U)), U)
    l = np.where(np.array(MAP_CATS) == 1, l1, r.uniform(0.0, 0.2, len(MAP_CATS)))
    assert (hm.length_scale(l)[hm.fixed_cols] == 1.0).all() and len(hm.fixed_cols) == 2
    told = _codes(r, 50, MAP_CATS)
    cand = np.asarray(sp.inverse_transform(U), dtype=np.float64)
    Kh = H.kernel(cand, told, l)
    Km = O.kernel_matrix(U, sp.transform(told.tolist()), hm.length_scale(l), kind="rbf")
    assert (np.abs(Km - Kh) <= 1e-15 * Kh).all()
    assert (hm.grad(np.ones(sp.transformed_n_dims))[np.array(MAP_CATS) == 1] == 0).all()


# ---- validation ------------------------------------------------------------------------------------------------------------
def test_optimizer_refuses_without_a_device():
    """Every refusal happens in the constructor; no engine exists before the first model-based ask."""
    cats = [Categorical(["a", "b", "c"], "opt"), Categorical([16, 32], "batch")]
    o = Optimizer(cats, kernel="hamming")
    assert o._engine is None and o._default_ls() == 1.0
    Optimizer(cats, kernel="hamming", theta_fit="skopt", random_state=2)
    for extra, word in (([Real(0.0, 1.0, "lr")], "lr"), ([Integer(1, 8, "layers")], "layers")):
        with pytest.raises(ValueError, match=word):
            Optimizer(cats + extra, kernel="hamming")
    for kw, word in ((dict(theta_grid=3), "theta_grid"), (dict(theta_search=2), "theta_search"), (dict(theta_fit="lbfgs"), "lbfgs"),
                     (dict(theta_fit="skopt", length_scale=0.5), "length_scale")):
        with pytest.raises(ValueError, match=word):
            Optimizer(cats, kernel="hamming", **kw)


def test_skopt_fit_drives_the_mapped_engine_calls():
    """The Optimizer's batched θ evaluations on a stand-in engine: each θ reaches lml_grad_batch as mapped column length scales
    of an RBF engine, and the fit the Optimizer reports is the oracle's, l_j and all."""
    c = CASES["mixed_d3_n100"]
    sp = space_of(c["categories"])
    hm = HM.HammingMap(sp)
    Xt = sp.transform(c["X"].tolist())

    class Stand:
        kernel, scratch_limit = "rbf", 1 << 30
        lml_grad_lane_bytes = staticmethod(lambda N, D, P: 1 << 20)

        def lml_grad_batch(self, X, y, thetas):
            out = [O.lml_and_grad(X, y, kind=self.kernel, length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
                   for th in thetas]
            return np.array([v for v, _ in out]), np.stack([g for _, g in out])

    res = TF.fit(TF.engine_batch_fn(Stand(), Xt, c["y"], hamming=hm), hm.n_dims, int(c["seed"]), 2, ls_bounds=HM.LS_BOUNDS)
    ref = H.skopt_fit(c["X"], c["y"], seed=int(c["seed"]))
    assert abs(res.lml - ref["lml"]) <= 1e-9 * abs(ref["lml"])
    assert np.abs(res.theta - ref["theta"]).max() <= 1e-5


# ---- gRPC ------------------------------------------------------------------------------------------------------------------
def categorical_experiment(settings=None, extra=(), name="ham-1"):
    """An Experiment over categorical and discrete lists (plus ``extra`` (name, type, min, max) parameters)."""
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "bayesianoptimization"
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, values in (("optimizer", api.CATEGORICAL, ["sgd", "adam", "rmsprop"]), ("batch", api.DISCRETE, ["16", "32", "64"]),
                                 ("bn", api.CATEGORICAL, ["on", "off"])):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        p.feasible_space.list.extend(values)
    for pname, ptype, lo, hi in extra:
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, ptype
        p.feasible_space.min, p.feasible_space.max = str(lo), str(hi)
    return e


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([SkoptService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _validate(stub, exp):
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))


def _refused(stub, exp, words, rpc="validate"):
    with pytest.raises(grpc.RpcError) as ei:
        if rpc == "validate":
            _validate(stub, exp)
        else:
            stub.GetSuggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=1))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    for w in words:
        assert w in ei.value.details(), ei.value.details()


def test_hamming_is_accepted_on_categorical_spaces(stub):
    _validate(stub, categorical_experiment({"kernel": "hamming"}))
    _validate(stub, categorical_experiment({"kernel": "hamming", "theta_fit": "skopt", "theta_restarts": 1}))
    _validate(stub, categorical_experiment({"kernel": "hamming", "length_scale": 0.5, "acq_func": "LCB"}))


@pytest.mark.parametrize("pname,ptype", [("lr", api.DOUBLE), ("layers", api.INT)])
@pytest.mark.parametrize("rpc", ["validate", "get"])
def test_mixed_spaces_are_refused_naming_the_parameter(stub, pname, ptype, rpc):
    _refused(stub, categorical_experiment({"kernel": "hamming"}, extra=[(pname, ptype, 1, 8)]), ["hamming", pname], rpc)


@pytest.mark.parametrize("knob,value", [("theta_grid", 3), ("theta_search", 2), ("theta_fit", "lbfgs")])
def test_hamming_refuses_one_hot_length_scale_searches(stub, knob, value):
    _refused(stub, categorical_experiment({"kernel": "hamming", knob: value}), [knob, "hamming"])


@pytest.mark.parametrize("est", ["RF", "ET"])
def test_tree_estimators_still_refuse_kernel(stub, est):
    _refused(stub, categorical_experiment({"base_estimator": est, "kernel": "hamming"}), ["kernel", est])
    _refused(stub, categorical_experiment({"kernel": "laplace"}), ["kernel"])
