"""GPU: CMA-ES with Margin (kbo_cma_set_margin, cma_margin_kernel) and `cmaes` with `with_margin: true`.

* Resynchronised parity at (D, λ) = (10, 10) and (128, 4096) with half the dimensions discrete (level tables, binary,
  uneven lists and an arithmetic range): every generation the samples are the oracle's encoding of m + σ·(A∘y) on the
  GPU's own state, the A-scaled mean step matches the oracle's, and the GPU's margin correction equals
  `cma_margin_oracle.margin_step` applied to the GPU's own pre-correction state to 1e-12 relative (Φ and Φ⁻¹ are CUDA's
  normcdf / normcdfinv against SciPy's ndtr and χ²₁.isf), widened in the side case by the conditioning of χ = Φ⁻¹(1 − q):
  a tail q carries a relative rounding of a few ε, which moves χ by 4ε·q/φ(χ), and A_j by that over χ_lo + χ_up.  Once
  s_j is far above the level spacing both χ are near 0 and this term passes 1e-12 (1.5e-12 seen at D = 128, generation 2).  A dimension whose case test lands within 1e-9 of its threshold
  on the oracle's side may take the other branch and is not compared (counted, at most 1 in 1000).  Both branches fire.
* The invariant holds on the device state after every tell.
* `set_margin({})` leaves 200 generations bit-identical to the parent commit's margin-free run.
* Restarts reset A and recompute the default α; gRPC Experiments over mixed int / discrete / double spaces hand out valid
  values and complete generations through duplicates and failed trials.
* The integer ellipsoid of tests/test_cma_margin_oracle.py, on the GPU with the same seeds and draws.
"""
import numpy as np
import pytest
import torch
from scipy.stats import norm

from oracle import cma_margin_oracle as M
from oracle import cma_oracle as O
from tests.test_cma_margin_oracle import SEEDS, integer_ellipsoid_runs
from tests.test_gpu_cma_restart import PARENT_DIGESTS, _cost_tool

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
SEEN = set()
SKIPPED = [0, 0]          # (dimension-generations not compared, compared)
WORST = [0.0, 0.0]        # (largest error / tolerance, largest conditioning term)


def _es(D, lam, seed=0, mean=0.5, sigma=1.0 / 6.0):
    from kubeflow_b200.cmaes import CmaEs
    return CmaEs(np.full(D, mean), sigma, popsize=lam, seed=seed)


def _dims(D):
    kinds = [np.linspace(0, 1, 5), np.array([0.0, 1.0]), (0.0, 1.0 / 5000, 5001), np.array([0.0, 0.1, 0.15, 0.6, 1.0]),
             np.arange(11) / 10.0]
    return {j: kinds[(j // 2) % len(kinds)] for j in range(0, D, 2)}


def _near_branch(m, A, sigma, c_diag, dim, alpha):
    l_lo, l_up = M.limits(dim, m)
    p_lo, p_up = M.tails(m, sigma * A * np.sqrt(c_diag), l_lo, l_up)
    hi, lo = max(p_lo, p_up), min(p_lo, p_up)
    return abs(hi - 0.5) <= 1e-9 or abs(lo - alpha) <= 1e-9 * alpha


def _parity(D, lam, gens, seed):
    dims = _dims(D)
    r = np.random.default_rng(seed)
    xs = M.encode(dims, r.uniform(0.1, 0.9, D))
    w = 10.0 ** (2 * np.arange(D) / (D - 1))
    f = lambda X: ((np.clip(X, 0, 1) - xs) ** 2 * w).sum(1)
    es = _es(D, lam, seed)
    es.set_margin(dims)
    ms = es.margin_state()
    alpha = ms["alpha"]
    assert alpha == 1.0 / (D * lam) and np.array_equal(ms["A"], np.ones(D))
    p = O.CmaParams(D, lam)
    cases = set()
    for g in range(gens):
        A0 = es.margin_state()["A"]
        z = r.standard_normal((lam, D))
        X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
        st = es.state(with_Y=True)
        x_raw = st["mean"] + st["sigma"] * (A0 * st["Y"])
        cont = [j for j in range(D) if j not in dims]
        np.testing.assert_allclose(X[:, cont], x_raw[:, cont], rtol=4 * EPS, atol=4 * EPS * st["sigma"] * np.abs(st["Y"]).max())
        enc = M.encode(dims, x_raw)
        for j, dim in dims.items():
            # a raw coordinate within a few ulp of a threshold may round to either side of it (DFMA against NumPy)
            near = np.abs(x_raw[:, j] - M.threshold(dim, np.clip(M.rank(dim, x_raw[:, j], False) - 1, 0, M.count(dim) - 2))) < 1e-14
            near |= np.abs(x_raw[:, j] - M.threshold(dim, np.minimum(M.rank(dim, x_raw[:, j], False), M.count(dim) - 2))) < 1e-14
            assert np.array_equal(X[~near, j], enc[~near, j]), f"generation {g} dim {j}: encoding"
        fx = f(X)
        es.tell(fx)
        new, mg = es.state(), es.margin_state()
        # the A-scaled mean step from the pre-tell state
        order = np.lexsort((np.arange(lam), fx))
        y_w = (st["Y"][order][:p.mu] * p.weights[:p.mu, None]).sum(0)
        want_pre = st["mean"] + p.cm * st["sigma"] * (A0 * y_w)
        # y_w is a sum of μ terms, in 8 fixed-order partial sums on the device and pairwise in NumPy: 16ε of Σ|w_i y_i|
        # covers the √(μ/8) = 16 rounding walk at μ = 2048
        step_abs = p.cm * st["sigma"] * A0 * (np.abs(st["Y"][order][:p.mu]) * p.weights[:p.mu, None]).sum(0)
        tol = 4 * EPS * np.linalg.norm(want_pre) + 16 * EPS * np.linalg.norm(step_abs)
        assert np.linalg.norm(mg["mean_before"] - want_pre) <= tol, f"generation {g}: mean step"
        # the margin correction on the GPU's own pre-correction state
        c_diag = np.diag(new["C"])
        info = {}
        m_ref, A_ref, cs = M.margin_step(mg["mean_before"], A0, new["sigma"], c_diag, dims, alpha, info)
        assert np.array_equal(new["mean"][cont], mg["mean_before"][cont]) and np.array_equal(mg["A"][cont], np.ones(len(cont)))
        for j in dims:
            if _near_branch(mg["mean_before"][j], A0[j], new["sigma"], c_diag[j], dims[j], alpha):
                SKIPPED[0] += 1
                continue
            SKIPPED[1] += 1
            kappa = 0.0
            if j in info:
                q_lo, q_up, chi_lo, chi_up = info[j]
                kappa = 4 * EPS * (q_lo / norm.pdf(chi_lo) + q_up / norm.pdf(chi_up)) / (chi_lo + chi_up)
            l_lo, l_up = M.limits(dims[j], mg["mean_before"][j])
            tol_m, tol_A = 1e-12 * abs(m_ref[j]) + kappa * (l_up - l_lo), (1e-12 + kappa) * abs(A_ref[j])
            err_m, err_A = abs(new["mean"][j] - m_ref[j]), abs(mg["A"][j] - A_ref[j])
            WORST[0], WORST[1] = max(WORST[0], err_m / tol_m, err_A / tol_A), max(WORST[1], kappa)
            assert err_m <= tol_m, f"generation {g} dim {j} ({cs[j]}): m {new['mean'][j]!r} oracle {m_ref[j]!r}, kappa {kappa:.3g}"
            assert err_A <= tol_A, f"generation {g} dim {j} ({cs[j]}): A {mg['A'][j]!r} oracle {A_ref[j]!r}, kappa {kappa:.3g}"
            cases.add(cs[j])
        bad = M.invariant_violations(new["mean"], mg["A"], new["sigma"], c_diag, dims, alpha, cs, mg["mean_before"])
        assert not bad, f"generation {g}: {bad}"
    es.close()
    SEEN.update(cases)
    return cases


@pytest.mark.parametrize("D,lam,gens", [(10, 10, 400), (128, 4096, 60)])
def test_margin_step_matches_the_oracle_on_the_gpu_state(D, lam, gens):
    cases = _parity(D, lam, gens, seed=D)
    print(f"\nMEASURED margin parity D={D} lam={lam}: cases {sorted(cases)}, not compared {SKIPPED[0]} of {sum(SKIPPED)}, "
          f"worst error/tolerance {WORST[0]:.3g}, largest conditioning term {WORST[1]:.3g}")


def test_both_branches_fired_and_few_were_skipped():
    assert {"edge-moved", "side"} <= SEEN, SEEN
    assert SKIPPED[0] * 1000 <= sum(SKIPPED)


@pytest.mark.parametrize("D,lam", list(PARENT_DIGESTS))
def test_all_continuous_margin_is_bit_identical_to_the_parent(D, lam):
    es = _es(D, lam, seed=7, mean=3.0, sigma=2.0)
    es.set_margin({})
    got = _cost_tool().digest(es)
    es.close()
    assert got == PARENT_DIGESTS[(D, lam)]


@pytest.mark.parametrize("alpha", [None, 0.03])
def test_restart_resets_A_and_the_default_alpha(alpha):
    D, lam = 6, 8
    es = _es(D, lam, seed=2)
    es.set_margin(_dims(D), alpha)
    for _ in range(30):
        es.tell(((es.ask().cpu().numpy() - 0.31) ** 2).sum(1))
    ms = es.margin_state()
    assert not np.array_equal(ms["A"], np.ones(D)) and ms["alpha"] == (alpha or 1.0 / (D * lam))
    for lam2 in (16, 5):                           # IPOP doubles λ; a BIPOP small run shrinks it
        es.restart(lam2, np.full(D, 0.4), 0.1)
        ms = es.margin_state()
        assert np.array_equal(ms["A"], np.ones(D)) and ms["alpha"] == (alpha or 1.0 / (D * lam2))
        X = es.ask().cpu().numpy()
        assert X.shape == (lam2, D) and np.array_equal(X, M.encode(_dims(D), X))
        es.tell((X ** 2).sum(1))
    es.close()


@pytest.mark.parametrize("strategy", ["ipop", "bipop"])
def test_grpc_restarts_with_margin(strategy, monkeypatch):
    from kubeflow_b200 import cmaes as cm
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from tests.test_grpc_service import add_trial
    seen = []
    orig = cm.CmaEs.restart

    def spy(self, lam, mean, sigma):
        orig(self, lam, mean, sigma)
        seen.append((lam, self.margin_state()))
    monkeypatch.setattr(cm.CmaEs, "restart", spy)
    e = _mixed_experiment(f"margin-{strategy}", {"with_margin": "true", "restart_strategy": strategy, "random_state": 3})
    svc = CmaesService()
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=0)
    svc.get_suggestions(req)
    k = 0
    while len(seen) < 2:                     # a constant loss stops each run by TOLFUN after term generations
        req.current_request_number = len(svc._exps[e.name].queue)
        for pa in svc.get_suggestions(req).parameter_assignments:
            a = {x.name: x.value for x in pa.assignments}
            assert _valid(a), a
            add_trial(req, f"t{k}", a, 1.5)
            k += 1
        req.current_request_number = 0
        svc.get_suggestions(req)
        assert k < 20000, "no restart"
    for lam, ms in seen:
        assert np.array_equal(ms["A"], np.ones(4)) and ms["alpha"] == 1.0 / (4 * lam)
    svc._exps[e.name].es.close()


def _mixed_experiment(name, settings):
    from kubeflow_b200.suggestion import api_pb as api
    from tests.test_grpc_service import make_experiment
    e = make_experiment("cmaes", settings, name=name)
    del e.spec.parameter_specs.parameters[:]
    for pname, kind, lo, hi, step, values in (("layers", api.INT, "1", "6", None, None), ("lr", api.DOUBLE, "0.001", "0.1", None, None),
                                              ("batch", api.DISCRETE, None, None, None, ["16", "32", "64", "128", "256"]),
                                              ("epochs", api.INT, "2", "20", "2", None)):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, kind
        if values:
            p.feasible_space.list.extend(values)
        else:
            p.feasible_space.min, p.feasible_space.max = lo, hi
            if step:
                p.feasible_space.step = step
    return e


def _valid(a):
    return (a["layers"] in [str(i) for i in range(1, 7)] and 0.001 <= float(a["lr"]) <= 0.1
            and a["batch"] in ("16", "32", "64", "128", "256") and a["epochs"] in [str(i) for i in range(2, 21, 2)])


def test_grpc_experiment_with_duplicates_and_failed_trials():
    import grpc
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    from tests.test_grpc_service import add_trial
    svc = CmaesService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    stub = SuggestionStub(ch)
    e = _mixed_experiment("margin-grpc", {"with_margin": "true", "popsize": 8, "random_state": 1})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=e))
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=0)
    k, dup_gens = 0, 0
    loss = lambda a: (int(a["layers"]) - 4) ** 2 + (np.log2(int(a["batch"])) - 6) ** 2 + (int(a["epochs"]) - 10) ** 2 / 4 \
        + (np.log10(float(a["lr"])) + 2) ** 2
    for gen in range(25):
        st = svc._exps.get(e.name)
        req.current_request_number = 8
        rep = stub.GetSuggestions(req)
        pts = [{x.name: x.value for x in pa.assignments} for pa in rep.parameter_assignments]
        assert len(pts) == 8 and all(_valid(a) for a in pts), pts
        dup_gens += len({tuple(sorted((n, v) for n, v in a.items() if n != "lr")) for a in pts}) < 8
        st = svc._exps[e.name]
        g0 = st.es.state()["generation"]
        for i, a in enumerate(pts):          # one failed trial per generation: its sample is handed out again
            add_trial(req, f"t{k}", a, loss(a), condition=api.FAILED if i == 3 else api.SUCCEEDED)
            k += 1
        req.current_request_number = 1
        rep = stub.GetSuggestions(req)
        again = {x.name: x.value for x in rep.parameter_assignments[0].assignments}
        assert again == pts[3]
        add_trial(req, f"t{k}", again, loss(again))
        k += 1
        req.current_request_number = 0
        stub.GetSuggestions(req)
        assert svc._exps[e.name].es.state()["generation"] == g0 + 1, f"generation {gen} did not complete"
    assert dup_gens > 0                      # the integer levels repeat, so the by-index matching was exercised
    svc._exps[e.name].es.close()
    ch.close()
    server.stop(0)


def test_integer_ellipsoid_on_the_gpu_with_the_oracles_seeds():
    """The oracle's runs (same seeds and draws) on the GPU sampler: CMAwM reaches the optimum at least as often as the
    oracle's plain rounding, as on the CPU."""
    D, K, lam, gens = 6, 11, 10, 300
    hits = {}
    for margin in (True, False):
        n = 0
        for seed in SEEDS:
            r = np.random.default_rng(100 + seed)
            xs = r.integers(0, K, D)
            w = 10.0 ** (3 * np.arange(D) / (D - 1))
            es = _es(D, lam)
            if margin:
                es.set_margin({j: np.linspace(0, 1, K) for j in range(D)})
            best = np.inf
            for _ in range(gens):
                X = es.ask(torch.tensor(r.standard_normal((lam, D)), device="cuda")).cpu().numpy()
                fx = ((np.round(np.clip(X, 0, 1) * (K - 1)) - xs) ** 2 * w).sum(1)
                best = min(best, fx.min())
                if best == 0:
                    break
                es.tell(fx)
            es.close()
            n += best == 0
        hits[margin] = n
    oracle_rounding = integer_ellipsoid_runs(False)
    print(f"\nMEASURED GPU integer ellipsoid hits over {len(SEEDS)} seeds: with_margin {hits[True]}, rounding {hits[False]} "
          f"(oracle rounding {oracle_rounding})")
    assert hits[True] > oracle_rounding and hits[True] > hits[False]
