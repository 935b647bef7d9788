"""GPU: separable CMA-ES (kbo_sepcma_*; sepcma_update_kernel, sepcma_finish_kernel, sepcma_should_stop_kernel) and `cmaes`
with `use_separable_cma: true`.

* Resynchronised per-generation parity at (D, λ) ∈ {(2, 6), (10, 10), (128, 18), (128, 4096), (1000, 24), (4096, 28),
  (4096, 512)} on the sphere, a separable and a rotated ellipsoid of condition 1e6 and a noisy Rastrigin: every generation
  `sepcma_oracle.tell` is given the GPU's own pre-tell state and steps Y and the fitness, and m, σ, p_σ, p_c, C and d after
  the tell must match within the bounds of `_tolerances`; the worst error over its tolerance is printed per case.
* Stop flags equal `sepcma_oracle.should_stop` on the GPU's state after every tell, and each of the five bits fires.
* ask(z) is fma(σ, d∘z, m) bit for bit; the built-in sampler's moments; bit-for-bit replay; restarts; ABI refusals.
* gRPC Experiments at D = 200 and D = 1000 (past the full sampler's 128) complete their generations through failed and
  duplicated trials; IPOP / BIPOP restarts through the service.
* A (128, 4096) run from mean 3, σ 2 on Rastrigin stays finite: the rank-μ rate is capped there.
"""
import functools
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import cma_oracle as O
from oracle import cma_restart_oracle as R
from oracle import sepcma_oracle as S
from tests.test_gpu_cma_long import _philox_normals

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
SEEN = set()


def _es(D, lam, seed=0, mean=0.5, sigma=1.0 / 6.0):
    from kubeflow_b200.cmaes import SepCmaEs
    return SepCmaEs(np.full(D, mean) if np.isscalar(mean) else mean, sigma, popsize=lam, seed=seed)


@functools.lru_cache(maxsize=None)
def _rotation(D, seed):
    return np.linalg.qr(np.random.default_rng(seed).standard_normal((D, D)))[0]


def _objective(name, D, seed):
    r = np.random.default_rng(seed)
    xs = r.uniform(0.3, 0.7, D)
    s = 1e6 ** (np.arange(D) / max(D - 1, 1))
    if name == "sphere":
        return lambda X: ((X - xs) ** 2).sum(1)
    if name == "sep_ellipsoid":
        return lambda X: (((X - xs) ** 2) * s).sum(1)
    if name == "rot_ellipsoid":
        Q = _rotation(D, seed)
        return lambda X: ((((X - xs) @ Q.T) ** 2) * s).sum(1)
    return lambda X: O.rastrigin((X - xs) * 10.24) + r.standard_normal(len(X))


def _load(st, lam):
    ref = S.SepState(st["mean"], st["sigma"], lam)
    ref.C, ref.p_sigma, ref.pc, ref.g = st["C"].copy(), st["p_sigma"].copy(), st["pc"].copy(), st["generation"]
    return ref


def _gamma(n):
    return n * EPS / (1 - n * EPS)


def _tolerances(st, Y, fx, ref, h):
    """Per-component bounds on |GPU − oracle| after one tell from the same state, assembled by the triangle inequality from
    the operation counts (each side's rounding counted once, so the sums carry 2γ):
      weights: ln((λ+1)/2) − ln i cancels, so each weight is off by up to 4ε·w_1 (the largest), host libm against NumPy;
      y_w,j = Σ_{r<μ} w_r y_r,j:  δy_w,j = 2γ_μ·Σ w_r|y_r,j| + 4ε·w_1·Σ|y_r,j|;  Σ w y² likewise with γ_{μ+1};
      m_j: σ·δy_w,j + 4ε(|m_j| + σ|y_w,j|);  p_σ,j: k_σ·δy_w,j/d_j + 8ε(|(1−c_σ)p_σ,j| + k_σ|y_w,j|/d_j);
      ‖p_σ‖² over D terms: 2γ_D‖p_σ‖² + 2‖p_σ‖‖δp_σ‖, so δ‖p_σ‖ is that over 2‖p_σ‖;
      σ = σ₀·exp(u), u = (c_σ/d_σ)(‖p_σ‖/χ_n − 1): relative (c_σ/d_σ)·δ‖p_σ‖/χ_n, plus 16ε(1 + |u| + (c_σ/d_σ)‖p_σ‖/χ_n)
        for the host constants, exp's ulp on each side and the products;
      p_c,j: k_c·δy_w,j + 8ε(|(1−c_c)p_c,j| + k_c|y_w,j|) (h_σ resynchronised);
      C_j: 2c1|p_c,j|δp_c,j + cμ·δ(Σ w y²)_j + 8ε(|a·C_j| + c1 p_c,j² + cμ Σ w y²_j) + 8ε·C_j for a's constants;
      d_j = √C_j: δC_j/(2d_j) + 2ε·d_j.
    Each bound is then doubled for the rounding counts left out."""
    SAFETY = 2.0
    p, lam = ref.p, len(fx)
    order = np.lexsort((np.arange(lam), np.asarray(fx)))
    Ys = np.asarray(Y)[order][:p.mu]
    w = p.weights[:, None]
    d0 = S.sqrt_c(st["C"])
    A = np.abs(Ys)
    yw = (Ys * w).sum(0)
    wy2 = (Ys * Ys * w).sum(0)
    e_yw = 2 * _gamma(p.mu) * (A * w).sum(0) + 4 * EPS * p.weights[0] * A.sum(0)
    e_wy2 = 2 * _gamma(p.mu + 1) * wy2 + 4 * EPS * p.weights[0] * (A * A).sum(0)
    s0 = st["sigma"]
    tol = {}
    tol["mean"] = s0 * e_yw + 4 * EPS * (np.abs(st["mean"]) + s0 * np.abs(yw))
    ks = np.sqrt(p.c_sigma * (2 - p.c_sigma) * p.mu_eff)
    tol["p_sigma"] = ks * e_yw / d0 + 8 * EPS * (np.abs((1 - p.c_sigma) * st["p_sigma"]) + ks * np.abs(yw) / d0)
    nps = np.linalg.norm(ref.p_sigma)
    e_n2 = 2 * _gamma(p.n) * nps ** 2 + 2 * nps * np.linalg.norm(tol["p_sigma"])
    e_n = e_n2 / (2 * nps) if nps > 0 else np.sqrt(e_n2)
    r = p.c_sigma / p.d_sigma
    u = r * (nps / p.chi_n - 1)
    tol["sigma"] = (r * e_n / p.chi_n + 16 * EPS * (1 + abs(u) + r * nps / p.chi_n)) * ref.sigma
    kc = h * np.sqrt(p.cc * (2 - p.cc) * p.mu_eff)
    tol["pc"] = kc * e_yw + 8 * EPS * (np.abs((1 - p.cc) * st["pc"]) + kc * np.abs(yw))
    a = 1 + p.c1 * (1 - h) * p.cc * (2 - p.cc) - p.c1 - p.cmu
    tol["C"] = (2 * p.c1 * np.abs(ref.pc) * tol["pc"] + p.cmu * e_wy2
                + 8 * EPS * (np.abs(a * st["C"]) + p.c1 * ref.pc ** 2 + p.cmu * wy2) + 8 * EPS * np.abs(st["C"]))
    dn = S.sqrt_c(ref.C)
    tol["d"] = tol["C"] / (2 * dn) + 2 * EPS * dn
    return {k: SAFETY * v for k, v in tol.items()}


def _ratios(got, ref, tol):
    out = {}
    for k, want in (("mean", ref.mean), ("p_sigma", ref.p_sigma), ("pc", ref.pc), ("C", ref.C), ("d", S.sqrt_c(ref.C)),
                    ("sigma", ref.sigma)):
        err = np.abs(np.asarray(got[k]) - want)
        t = np.asarray(tol[k])
        rat = np.where(t > 0, err / np.where(t > 0, t, 1), np.where(err == 0, 0.0, np.inf))
        out[k] = float(np.max(rat))
    return out


SHAPES = [(2, 6, 300), (10, 10, 300), (128, 18, 150), (128, 4096, 30), (1000, 24, 100), (4096, 28, 60), (4096, 512, 15)]


@pytest.mark.parametrize("name", ["sphere", "sep_ellipsoid", "rot_ellipsoid", "noisy_rastrigin"])
@pytest.mark.parametrize("D,lam,gens", SHAPES, ids=[f"D{d}-lam{l}" for d, l, _ in SHAPES])
def test_resynchronised_parity(D, lam, gens, name):
    f = _objective(name, D, seed=D)
    es = _es(D, lam, seed=D)
    r = np.random.default_rng(D + 1)
    worst, where, hflips = 0.0, "", 0
    for g in range(gens):
        z = r.standard_normal((lam, D))
        X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
        st = es.state(with_Y=True)
        fx = f(X)
        es.tell(fx)
        got = es.state()
        probe = S.tell(_load(st, lam), st["Y"], fx)
        nps = np.linalg.norm(probe.p_sigma)
        hl, thr = S.h_left(_load(st, lam), nps), S.h_threshold(probe.p)
        cands = [1.0 if hl < thr else 0.0]
        if abs(hl - thr) <= 1e-12 * thr:                 # h_σ within rounding of its threshold: either branch
            cands.append(1.0 - cands[0])
        best = None
        for h in cands:
            ref = S.tell(_load(st, lam), st["Y"], fx, h_sigma=h)
            ratio = _ratios(got, ref, _tolerances(st, st["Y"], fx, ref, h))
            if best is None or max(ratio.values()) < max(best[0].values()):
                best = (ratio, h)
        ratio, h = best
        hflips += h != cands[0]
        k = max(ratio, key=ratio.get)
        if ratio[k] > worst:
            worst, where = ratio[k], f"generation {g} {k}"
        assert max(ratio.values()) <= 1.0, f"{name} D={D} lam={lam} generation {g}: error/tolerance {ratio}"
    es.close()
    print(f"\nMEASURED sepcma parity {name} D={D} lam={lam}: worst error/tolerance {worst:.3g} at {where}; "
          f"sigma {got['sigma']:.4g}; h_sigma alternatives taken {hflips}")


# ------------------------------------------------------------------------------------------------ termination test
def _drive(D, lam, f, gens, mean=0.5, sigma=1.0 / 6.0, seed=0, until=None):
    es = _es(D, lam, seed, mean, sigma)
    tolx, term = R.tolx(sigma), R.funhist_term(D, lam)
    hist = np.zeros(2 * term)
    flags, h0, t0 = es.stop_flags()
    assert flags == 0 and t0 == term and not h0.any()
    seen = 0
    for _ in range(gens):
        fx = f(es.ask().cpu().numpy())
        es.tell(fx)
        st = es.state()
        R.record(hist, st["generation"], term, fx)
        flags, gh, _ = es.stop_flags()
        assert np.array_equal(gh, hist, equal_nan=True)
        want = S.should_stop(st["mean"], st["sigma"], st["C"], st["pc"], st["d"], gh, st["generation"], term, tolx)
        assert flags == want, f"generation {st['generation']}: GPU flags {flags:#x}, oracle on the GPU state {want:#x}"
        assert not flags & R.NOEFFECTAXIS
        SEEN.update(b for b, v in R.BITS.items() if flags & v)
        seen |= flags
        if until is not None and flags & until:
            break
    es.close()
    return seen


def test_tolxup_from_a_huge_sigma():
    assert _drive(4, 8, O.sphere, 3, sigma=1e5) & R.TOLXUP


def test_noeffect_coord_at_mean_1e17():
    assert _drive(4, 8, lambda X: ((X - 1e17) ** 2).sum(1), 5, mean=1e17) & R.NOEFFECTCOORD


def test_tolfun_on_constant_fitness():
    D, lam = 3, 7
    assert _drive(D, lam, lambda X: np.full(len(X), 2.5), R.funhist_term(D, lam) + 1) & R.TOLFUN


def test_tolx_on_a_long_sphere_run():
    xs = np.array([0.3, 0.6])
    assert _drive(2, 6, lambda X: 1e20 * ((X - xs) ** 2).sum(1), 2000, until=R.TOLX) & R.TOLX


def test_conditioncov_on_an_ill_conditioned_ellipsoid():
    s, xe = np.array([1.0, 1e30]), np.array([0.3, 0.0])
    assert _drive(2, 6, lambda X: (((X - xe) ** 2) * s).sum(1), 3000, until=R.CONDITIONCOV) & R.CONDITIONCOV


@pytest.mark.parametrize("D,lam", [(5, 9), (4096, 28)])
def test_flags_along_a_run_with_nan_and_inf_fitness(D, lam):
    r = np.random.default_rng(3)

    def f(X):
        v = O.sphere(X - 0.4)
        k = r.integers(0, len(v), 2)
        v[k] = (np.nan, np.inf) if r.random() < 0.5 else (-np.inf, np.nan)
        return v
    _drive(D, lam, f, 30)


def test_every_bit_but_noeffectaxis_fired_somewhere_in_this_module():
    want = set(R.BITS) - {"NOEFFECTAXIS"}
    assert SEEN == want, f"never fired: {sorted(want - SEEN)}"


# ------------------------------------------------------------------------------------------------ sampler
def test_large_population_run_stays_finite():
    # at (128, 4096) the recalled rank-μ rate is about 5.0 and is capped at 1 − c1 − 1e-8; uncapped, C turned negative
    es = _es(128, 4096, seed=7, mean=3.0, sigma=2.0)
    for _ in range(300):
        X = es.ask()
        es.tell(10.0 * X.shape[1] + (X * X - 10.0 * torch.cos(2 * np.pi * X)).sum(1))
    st = es.state()
    assert np.isfinite(st["sigma"]) and (st["C"] > 0).all() and np.isfinite(st["C"]).all() and np.isfinite(st["mean"]).all()
    es.close()


def test_ask_with_z_is_the_fused_step():
    D, lam = 10, 10
    es = _es(D, lam, seed=4)
    f = _objective("sep_ellipsoid", D, 4)
    for _ in range(20):
        es.tell(f(es.ask().cpu().numpy()))
    z = np.random.default_rng(9).standard_normal((lam, D))
    X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
    st = es.state(with_Y=True)
    assert np.array_equal(st["Y"], z * st["d"])
    want = np.array([[float(Fraction(st["sigma"]) * Fraction(float(y)) + Fraction(float(m))) for y, m in zip(row, st["mean"])]
                     for row in st["Y"]])
    assert np.array_equal(X, want)
    es.close()


def test_builtin_sampler_moments():
    D, lam = 1000, 1000
    es = _es(D, lam, seed=12, mean=0.0, sigma=1.0)
    Z = es.ask().cpu().numpy()                     # d = 1, m = 0, σ = 1: x = z
    n = Z.size
    assert abs(Z.mean()) < 5 / np.sqrt(n) and abs(Z.var() - 1) < 5 * np.sqrt(2 / n)
    assert abs((Z ** 3).mean()) < 5 * np.sqrt(15 / n) and abs((Z ** 4).mean() - 3) < 5 * np.sqrt(96 / n)
    np.testing.assert_allclose(Z.ravel(), _philox_normals(n, 12, 0), rtol=0, atol=1e-13)
    es.tell(O.sphere(Z - 0.1))
    X = es.ask().cpu().numpy()
    st = es.state()
    W = (X - st["mean"]) / (st["sigma"] * st["d"])
    assert abs(W.mean()) < 5 / np.sqrt(n) and abs(W.var() - 1) < 5 * np.sqrt(2 / n)
    es.close()


def test_free_running_run_replays_bit_for_bit():
    out = []
    for _ in range(2):
        es = _es(300, 16, seed=5)
        f = _objective("noisy_rastrigin", 300, 5)
        for _ in range(40):
            es.tell(f(es.ask().cpu().numpy()))
        out.append((es.state(with_Y=True), es.stop_flags()))
        es.close()
    (a, fa), (b, fb) = out
    for k in ("mean", "sigma", "C", "d", "p_sigma", "pc", "Y", "generation"):
        assert np.array_equal(a[k], b[k]), k
    assert fa[0] == fb[0] and np.array_equal(fa[1], fb[1])


_STATE_KEYS = ("mean", "sigma", "C", "p_sigma", "pc", "d", "generation")


@pytest.mark.parametrize("D,lam,lam2", [(10, 10, 20), (1000, 24, 6), (4096, 28, 8192)])
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
    es.restart(12, np.zeros(D), 1.0)                       # d = 1, m = 0, σ = 1: x = z exactly
    X = es.ask().cpu().numpy()
    np.testing.assert_allclose(X.ravel(), _philox_normals(D * 12, seed, 4), rtol=0, atol=1e-13)
    es.close()


def test_abi_refusals():
    from kubeflow_b200._lib import KboError, KboInvalidArgument
    from kubeflow_b200.cmaes import CmaEs
    for D, lam in ((0, 8), (4097, 8), (10, 3), (10, 8193)):
        with pytest.raises(KboInvalidArgument):
            _es(D, lam)
    with pytest.raises(KboInvalidArgument):
        CmaEs(np.full(200, 0.5), 0.2)                       # the full sampler stops at D = 128
    es = _es(4096, 8)
    with pytest.raises(KboError) as e:
        es.tell(np.arange(8.0))                            # a tell before an ask
    assert e.value.code == -5
    with pytest.raises(KboInvalidArgument):
        es.restart(3, np.zeros(4096), 1.0)
    es.close()


# ------------------------------------------------------------------------------------------------ the service
def _wide(name, D, settings):
    from kubeflow_b200.suggestion import api_pb as api
    from tests.test_grpc_service import make_experiment
    e = make_experiment("cmaes", settings, name=name)
    del e.spec.parameter_specs.parameters[:]
    for i in range(D):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = f"x{i}", api.INT if i < 2 else api.DOUBLE
        p.feasible_space.min, p.feasible_space.max = ("1", "4") if i < 2 else ("-1", "1")
    return e


@pytest.mark.parametrize("D,gens", [(200, 12), (1000, 6)])
def test_grpc_experiment_past_the_full_limit_with_failed_and_duplicated_trials(D, gens):
    """Each generation: one trial FAILED (its sample is handed out again and completed), and one completed assignment reported
    again under a second trial name (a duplicate: no sample waits for it, so it is ignored).  The generation must complete
    exactly once per round."""
    import grpc

    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    from tests.test_grpc_service import add_trial
    svc = CmaesService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}", options=[("grpc.max_send_message_length", 256 << 20),
                                                              ("grpc.max_receive_message_length", 256 << 20)])
    stub = SuggestionStub(ch)
    e = _wide(f"sep-grpc-{D}", D, {"use_separable_cma": "true", "random_state": 1})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=e))
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=0)
    lam = 4 + int(3 * np.log(D))
    xs = np.random.default_rng(D).uniform(-0.5, 0.5, D)
    loss = lambda a: float(sum((float(a[f"x{i}"]) - xs[i]) ** 2 for i in range(D)))
    k = 0
    for gen in range(gens):
        req.current_request_number = lam
        pts = [{x.name: x.value for x in pa.assignments} for pa in stub.GetSuggestions(req).parameter_assignments]
        assert len(pts) == lam and all(-1.0 <= float(a["x5"]) <= 1.0 and a["x0"] in "1234" for a in pts)
        st = svc._exps[e.name]
        assert type(st.es).__name__ == "SepCmaEs"
        g0 = st.es.state()["generation"]
        for i, a in enumerate(pts):
            add_trial(req, f"t{k}", a, loss(a), condition=api.FAILED if i == 3 else api.SUCCEEDED)
            k += 1
        add_trial(req, f"t{k}", pts[0], loss(pts[0]))       # the duplicate
        k += 1
        req.current_request_number = 1
        again = {x.name: x.value for x in stub.GetSuggestions(req).parameter_assignments[0].assignments}
        assert again == pts[3]
        add_trial(req, f"t{k}", again, loss(again))
        k += 1
        req.current_request_number = 0
        stub.GetSuggestions(req)
        assert svc._exps[e.name].es.state()["generation"] == g0 + 1, f"generation {gen} did not complete"
    s = svc._exps[e.name].es.state()
    assert s["C"].shape == (D,) and np.isfinite(s["C"]).all()
    svc._exps[e.name].es.close()
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("strategy", ["ipop", "bipop"])
def test_grpc_restarts_on_the_schedule(strategy, monkeypatch):
    from kubeflow_b200 import cmaes as cm
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from tests.test_grpc_service import add_trial
    seen = []
    orig = cm.SepCmaEs.restart

    def spy(self, lam, mean, sigma):
        seen.append((self.stop_flags()[0], self.popsize, lam))
        orig(self, lam, mean, sigma)
    monkeypatch.setattr(cm.SepCmaEs, "restart", spy)
    e = _wide(f"sep-{strategy}", 6, {"use_separable_cma": "true", "restart_strategy": strategy, "random_state": 3})
    svc = CmaesService()
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=0)
    svc.get_suggestions(req)
    k = 0
    while len(seen) < 2:                     # a constant loss stops each run by TOLFUN after term generations
        req.current_request_number = len(svc._exps[e.name].queue)
        for pa in svc.get_suggestions(req).parameter_assignments:
            add_trial(req, f"t{k}", {x.name: x.value for x in pa.assignments}, 1.5)
            k += 1
        req.current_request_number = 0
        svc.get_suggestions(req)
        assert k < 20000, "no restart"
    for flags, lam_before, lam_after in seen:
        assert flags & R.TOLFUN
    if strategy == "ipop":
        assert seen[0][2] == 2 * seen[0][1] and seen[1][2] == 2 * seen[1][1]
    svc._exps[e.name].es.close()
