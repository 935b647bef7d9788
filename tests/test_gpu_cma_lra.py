"""GPU: CMA-ES with learning-rate adaptation (kbo_cma_set_lr_adapt; cma_lra_prep_kernel, cma_lra_kernel and
cma_lra_finish_kernel) and `cmaes` with `lr_adapt: true`.

* Resynchronised per-generation parity at (D, λ) ∈ {(2, 6), (10, 10), (128, 18), (128, 4096)} on the sphere, a rotated
  ellipsoid of condition 1e6 and a noisy Rastrigin: every generation `cma_lra_oracle.lra_tell` is given the GPU's own
  pre-tell state (`state(with_Y=True)` and `lr_state()`), its steps Y, ‖z‖² and the fitness, and m, σ, C, d, E, V and η
  after the tell must match.  The tolerances are derived below (`_tolerances`); the worst error over its tolerance is
  printed per shape.
* The first tell's η_m and η_Σ equal the closed forms to 4ε; a free-running run replays bit for bit;
  `set_lr_adapt(False)` reproduces the parent commit's 200-generation digests.
* IPOP and BIPOP with LRA: the state resets at every restart, λ changing or not, directly and through the service.
* gRPC Experiments with `lr_adapt: true` complete their generations through duplicates and failed trials.
"""
from decimal import Decimal

import numpy as np
import pytest
import torch

from oracle import cma_lra_oracle as L
from oracle import cma_oracle as O
from tests.test_cma_lra_oracle import ETA_M1, ETA_S1
from tests.test_gpu_cma_long import TOL_C, TOL_EIG, TOL_MEAN, TOL_ORTH, TOL_PS, TOL_SIGMA, _load
from tests.test_gpu_cma_restart import PARENT_DIGESTS, _cost_tool

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
WORST = {}


def _es(D, lam, seed=0, mean=0.5, sigma=1.0 / 6.0, lra=True):
    from kubeflow_b200.cmaes import CmaEs
    es = CmaEs(np.full(D, mean), sigma, popsize=lam, seed=seed)
    if lra:
        es.set_lr_adapt(True)
    return es


def _objective(name, D, seed):
    if name == "noisy_rastrigin":
        r = np.random.default_rng(seed)
        xs = r.uniform(0.3, 0.7, D)
        return lambda X: O.rastrigin((X - xs) * 10.24) + r.standard_normal(len(X))
    return O.objective(name, D, seed)[0]


def _lra_from(ls, D):
    lra = L.LraState(D)
    lra.E_mean, lra.E_Sigma = ls["E_mean"].copy(), ls["E_Sigma"].copy()
    lra.V_mean, lra.V_Sigma, lra.eta_mean, lra.eta_Sigma = ls["V_mean"], ls["V_Sigma"], ls["eta_mean"], ls["eta_Sigma"]
    return lra


def _reference(st, ls, fx, zn2, h_sigma=None):
    ref, lra = _load(st, len(fx)), _lra_from(ls, len(st["mean"]))
    L.lra_tell(ref, lra, st["Y"], fx, znorm2=zn2, h_sigma=h_sigma)
    return ref, lra


def _snr_error(E, V, dE, dV, beta):
    """|δSNR| from errors dE (in ‖E‖) and dV: SNR = N/Dn with N = ‖E‖² − c·V and Dn = V − ‖E‖², c = β/(2 − β).  Both
    are cancellations, so the errors of ‖E‖² and V are divided by Dn, not by either term: δN ≤ δ‖E‖² + c·δV and
    δDn ≤ δV + δ‖E‖², so δSNR ≤ (δN + |SNR|·δDn)/Dn, with a rounding of 4ε on each of ‖E‖² and V."""
    E2, c = E * E, beta / (2.0 - beta)
    den = V - E2
    if not den > 0:
        return 0.0
    dE2 = 2 * E * dE + dE * dE + 4 * EPS * E2
    dV = dV + 4 * EPS * V
    s = (E2 - c * V) / den
    return (dE2 + c * dV + abs(s) * (dV + dE2)) / den


def _tolerances(st, ls, ref, lra, fx, zn2, h):
    """Each bound, from what the plain tell is allowed (tests/test_gpu_cma_long.py: m′ to TOL_MEAN·ε, C′ to TOL_C·ε·√λ of
    ‖C′‖₂, σ′ to TOL_SIGMA·ε·κ with κ = cond(C)) and what the local transform costs:
      P = Σ^{-1/2} = B diag(1/d) Bᵀ/σ, ‖P‖₂ = 1/(σ·d_min).  The device's B is orthogonal to TOL_ORTH (its Jacobi stopping
        rule) and d_min² carries TOL_EIG·ε·‖C‖₂, so P is off by ρ_P = TOL_ORTH + TOL_EIG·ε·κ relative: about κ·ε.
      Δ̃m = P·Δm: error ‖P‖₂·(δΔm + ρ_P·‖Δm‖), δΔm = TOL_MEAN·ε·‖m′‖ + ε‖m‖.
      Δ̃Σ = P·ΔΣ·P/√2: error ‖P‖₂²·(δΔΣ + 2ρ_P·‖ΔΣ‖_F)/√2, δΔΣ = σ′²·(TOL_C·ε·√λ·D + 2·TOL_SIGMA·ε·κ)·‖C′‖₂ + 4ε‖σ²C‖_F.
      E ← (1 − β)E + βΔ̃ and V ← (1 − β)V + β‖Δ̃‖²: βδΔ̃ and β(2‖Δ̃‖δΔ̃ + δΔ̃²), plus 8ε of each.
      SNR: `_snr_error`, both cancellations.
      η: exp(min(γη, β)·clip(SNR/(αη) − 1)) has slope η·min(γη, β)/(αη) in the SNR inside the clip's linear range and 0
        outside it; the linear slope bounds both.  Plus 4ε.
      m = m_prev + η_m·Δm: η_m·δΔm + δη_m·‖Δm‖ + 4ε‖m‖.
      Σ = σ²C + η_Σ·ΔΣ: η_Σ·δΔΣ + δη_Σ·‖ΔΣ‖_F + 4ε‖Σ‖_F; then σ_det = exp(log det Σ/2D) moves by
        ‖δΣ‖_F/(2λ_min(Σ)) + TOL_EIG·ε·κ(Σ)/2 relative (each log λ_j by δλ_j/λ_j), σ = σ_det·η_m,prev/η_m by δη_m/η_m
        more, and C = Σ/σ_det² by ‖δΣ‖_F/‖Σ‖₂ + 2δσ_det/σ_det of ‖C‖₂; sorted d² against eigh of the oracle's C by D·δC
        + TOL_EIG·ε·‖C‖₂ (the Jacobi decomposition's own bound).
    These are first-order bounds assembled by the triangle inequality, each multiplied by SAFETY = 4 for the constants of
    the rounding counts left out (sums of D or D² terms, the tree orders)."""
    SAFETY = 4.0
    D, lam = len(st["mean"]), len(fx)
    m0, s0, C0 = st["mean"], st["sigma"], st["C"]
    ev0 = np.linalg.eigvalsh(C0)
    kappa = ev0[-1] / ev0[0]
    P2 = 1.0 / (s0 * np.sqrt(ev0[0]))
    rho_P = TOL_ORTH + TOL_EIG * EPS * kappa
    eta_prev_m = ls["eta_mean"]
    plain = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2, h_sigma=h)      # the plain step the blend starts from
    dm = plain.mean - m0
    dS = plain.sigma ** 2 * plain.C - s0 ** 2 * C0
    Cn2 = np.linalg.norm(plain.C, 2)
    e_dm = TOL_MEAN * EPS * np.linalg.norm(plain.mean) + EPS * np.linalg.norm(m0)
    e_dS = plain.sigma ** 2 * (TOL_C * EPS * np.sqrt(lam) * D + 2 * TOL_SIGMA * EPS * kappa) * Cn2 + 4 * EPS * np.linalg.norm(s0 ** 2 * C0)
    Pm = (st["B"] / st["d"]) @ st["B"].T / s0
    loc_m = np.linalg.norm(Pm @ dm)
    loc_S = np.linalg.norm(Pm @ dS @ Pm) / np.sqrt(2)
    e_lm = P2 * (e_dm + rho_P * np.linalg.norm(dm))
    e_lS = P2 * P2 * (e_dS + 2 * rho_P * np.linalg.norm(dS)) / np.sqrt(2)
    tol = {}
    tol["E_mean"] = L.BETA_MEAN * e_lm + 8 * EPS * np.linalg.norm(lra.E_mean)
    tol["E_Sigma"] = L.BETA_SIGMA * e_lS + 8 * EPS * np.linalg.norm(lra.E_Sigma)
    dVm = L.BETA_MEAN * (2 * loc_m * e_lm + e_lm ** 2)
    dVS = L.BETA_SIGMA * (2 * loc_S * e_lS + e_lS ** 2)
    tol["V_mean"] = dVm + 8 * EPS * lra.V_mean
    tol["V_Sigma"] = dVS + 8 * EPS * lra.V_Sigma
    d_snr_m = _snr_error(np.linalg.norm(lra.E_mean), lra.V_mean, tol["E_mean"], dVm, L.BETA_MEAN)
    d_snr_S = _snr_error(np.linalg.norm(lra.E_Sigma), lra.V_Sigma, tol["E_Sigma"], dVS, L.BETA_SIGMA)
    rate_m, rate_S = min(L.GAMMA * eta_prev_m, L.BETA_MEAN), min(L.GAMMA * ls["eta_Sigma"], L.BETA_SIGMA)
    tol["eta_mean"] = lra.eta_mean * rate_m * d_snr_m / (L.ALPHA * eta_prev_m) + 4 * EPS * lra.eta_mean
    tol["eta_Sigma"] = lra.eta_Sigma * rate_S * d_snr_S / (L.ALPHA * ls["eta_Sigma"]) + 4 * EPS * lra.eta_Sigma
    tol["mean"] = lra.eta_mean * e_dm + tol["eta_mean"] * np.linalg.norm(dm) + 4 * EPS * np.linalg.norm(ref.mean)
    Sigma = s0 ** 2 * C0 + lra.eta_Sigma * dS
    evS = np.linalg.eigvalsh(Sigma)
    e_Sig = lra.eta_Sigma * e_dS + tol["eta_Sigma"] * np.linalg.norm(dS) + 4 * EPS * np.linalg.norm(Sigma)
    d_sdet = e_Sig / (2 * evS[0]) + TOL_EIG * EPS * (evS[-1] / evS[0]) / 2
    tol["sigma"] = (d_sdet + tol["eta_mean"] / lra.eta_mean + 4 * EPS) * ref.sigma
    tol["C"] = (e_Sig / evS[-1] + 2 * d_sdet + 4 * EPS) * np.linalg.norm(ref.C, 2)
    tol["d2"] = D * tol["C"] + TOL_EIG * EPS * np.linalg.norm(ref.C, 2)
    return {k: SAFETY * v for k, v in tol.items()}


def _errors(got, gl, ref, lra):
    return dict(mean=np.linalg.norm(got["mean"] - ref.mean), sigma=abs(got["sigma"] - ref.sigma), C=np.abs(got["C"] - ref.C).max(),
                d2=np.abs(np.sort(got["d"] ** 2) - np.linalg.eigvalsh(ref.C)).max(),
                E_mean=np.linalg.norm(gl["E_mean"] - lra.E_mean), E_Sigma=np.linalg.norm(gl["E_Sigma"] - lra.E_Sigma),
                V_mean=abs(gl["V_mean"] - lra.V_mean), V_Sigma=abs(gl["V_Sigma"] - lra.V_Sigma),
                eta_mean=abs(gl["eta_mean"] - lra.eta_mean), eta_Sigma=abs(gl["eta_Sigma"] - lra.eta_Sigma))


SHAPES = [(2, 6, 300), (10, 10, 300), (128, 18, 100), (128, 4096, 30)]


@pytest.mark.parametrize("name", ["sphere", "ellipsoid1e6", "noisy_rastrigin"])
@pytest.mark.parametrize("D,lam,gens", SHAPES, ids=[f"D{d}-lam{l}" for d, l, _ in SHAPES])
def test_resynchronised_parity(D, lam, gens, name):
    f = _objective(name, D, seed=D)
    es = _es(D, lam, seed=D)
    r = np.random.default_rng(D + 1)
    worst, where, hflips = 0.0, "", 0
    for g in range(gens):
        z = r.standard_normal((lam, D))
        X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
        st, ls = es.state(with_Y=True), es.lr_state()
        fx = f(X)
        es.tell(fx)
        got, gl = es.state(), es.lr_state()
        zn2 = (z * z).sum(1)
        cands = [None]
        p = O.CmaParams(D, lam)
        probe = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2)
        h_left = np.linalg.norm(probe.p_sigma) / np.sqrt(1 - (1 - p.c_sigma) ** (2 * (st["generation"] + 1)))
        thr = (1.4 + 2 / (D + 1)) * p.chi_n
        kappa = np.linalg.cond(st["C"])
        if abs(h_left - thr) <= TOL_PS * EPS * kappa * h_left:     # h_σ within rounding of its threshold: either branch
            cands.append(0.0 if h_left < thr else 1.0)
        best = None
        for h in cands:
            ref, lra = _reference(st, ls, fx, zn2, h)
            tol = _tolerances(st, ls, ref, lra, fx, zn2, h)
            err = _errors(got, gl, ref, lra)
            ratio = {k: err[k] / tol[k] if tol[k] > 0 else (0.0 if err[k] == 0 else np.inf) for k in err}
            if best is None or max(ratio.values()) < max(best[0].values()):
                best = (ratio, err, tol, h)
        ratio, err, tol, h = best
        hflips += h is not None
        k = max(ratio, key=ratio.get)
        if ratio[k] > worst:
            worst, where = ratio[k], f"generation {g} {k}"
        for q in ratio:
            assert ratio[q] <= 1.0, f"{name} D={D} lam={lam} generation {g}: {q} error {err[q]:.3g} > tolerance {tol[q]:.3g} " \
                                    f"(eta {gl['eta_mean']:.4g}/{gl['eta_Sigma']:.4g}, cond(C) {kappa:.3g})"
    es.close()
    WORST[(D, lam, name)] = worst
    print(f"\nMEASURED lra parity {name} D={D} lam={lam}: worst error/tolerance {worst:.3g} at {where}; "
          f"eta_mean {gl['eta_mean']:.4g} eta_Sigma {gl['eta_Sigma']:.4g}; h_sigma alternatives taken {hflips}")


def test_first_tell_closed_forms():
    for D, lam in ((2, 6), (10, 10), (128, 18), (128, 4096)):
        es = _es(D, lam, seed=3)
        X = es.ask().cpu().numpy()
        es.tell(O.sphere(X - 0.3))
        ls = es.lr_state()
        es.close()
        for got, want in ((ls["eta_mean"], ETA_M1), (ls["eta_Sigma"], ETA_S1)):
            assert abs(Decimal(got) - want) <= 4 * Decimal(EPS) * want, (D, lam, got, want)


def test_free_running_run_replays_bit_for_bit():
    out = []
    for _ in range(2):
        es = _es(10, 10, seed=5)
        f = _objective("ellipsoid1e6", 10, 5)
        for _ in range(60):
            es.tell(f(es.ask().cpu().numpy()))
        out.append((es.state(with_Y=True), es.lr_state()))
        es.close()
    (a, la), (b, lb) = out
    for k in ("mean", "sigma", "C", "B", "d", "p_sigma", "pc", "Y"):
        assert np.array_equal(a[k], b[k]), k
    for k in la:
        assert np.array_equal(la[k], lb[k]), k
    assert la["eta_mean"] < 1.0


@pytest.mark.parametrize("D,lam", list(PARENT_DIGESTS))
def test_lr_adapt_off_is_bit_identical_to_the_parent(D, lam):
    es = _es(D, lam, seed=7, mean=3.0, sigma=2.0)       # turned on, then off: the plain path
    es.set_lr_adapt(False)
    got = _cost_tool().digest(es)
    es.close()
    assert got == PARENT_DIGESTS[(D, lam)]


def _fresh(ls, D):
    return (np.array_equal(ls["E_mean"], np.zeros(D)) and np.array_equal(ls["E_Sigma"], np.zeros((D, D)))
            and (ls["V_mean"], ls["V_Sigma"], ls["eta_mean"], ls["eta_Sigma"]) == (0.0, 0.0, 1.0, 1.0))


def test_restart_resets_the_lra_state():
    D, lam = 6, 8
    es = _es(D, lam, seed=2)
    for lam2 in (8, 16, 5):                             # same λ, IPOP's doubled λ, a BIPOP small run
        for _ in range(30):
            es.tell(O.sphere(es.ask().cpu().numpy() - 0.31) + np.random.default_rng(lam2).standard_normal(es.popsize))
        assert not _fresh(es.lr_state(), D)
        es.restart(lam2, np.full(D, 0.4), 0.1)
        assert _fresh(es.lr_state(), D) and es.popsize == lam2
        # the first tell of the new run is a first tell again
        es.tell(O.sphere(es.ask().cpu().numpy()))
        assert abs(Decimal(es.lr_state()["eta_mean"]) - ETA_M1) <= 4 * Decimal(EPS)
    es.close()


def test_abi_refusals():
    from kubeflow_b200._lib import KboError, KboInvalidArgument
    es = _es(4, 8, lra=False)
    with pytest.raises(KboError):
        es.lr_state()                                   # off
    es.set_margin({0: np.array([0.0, 0.5, 1.0])})
    with pytest.raises(KboInvalidArgument):
        es.set_lr_adapt(True)                           # not with a margin
    es.set_margin({})
    es.set_lr_adapt(True)
    with pytest.raises(KboInvalidArgument):
        es.set_margin({0: np.array([0.0, 1.0])})         # and no margin while it is on
    es.ask()
    with pytest.raises(KboError) as e:
        es.set_lr_adapt(False)                          # between an ask and its tell
    assert e.value.code == -5
    es.tell(np.arange(8.0))
    es.set_lr_adapt(True)                               # on again: a fresh state
    assert _fresh(es.lr_state(), 4)
    es.close()


def _experiment(name, settings):
    from kubeflow_b200.suggestion import api_pb as api
    from tests.test_grpc_service import make_experiment
    e = make_experiment("cmaes", settings, name=name)
    del e.spec.parameter_specs.parameters[:]
    for pname, kind, lo, hi in (("layers", api.INT, "1", "6"), ("lr", api.DOUBLE, "0.001", "0.1"), ("units", api.INT, "1", "4"),
                                ("dropout", api.DOUBLE, "0.0", "0.5")):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = pname, kind
        p.feasible_space.min, p.feasible_space.max = lo, hi
    return e


@pytest.mark.parametrize("strategy", ["ipop", "bipop"])
def test_grpc_restarts_reset_the_lra_state(strategy, monkeypatch):
    from kubeflow_b200 import cmaes as cm
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from tests.test_grpc_service import add_trial
    seen = []
    orig = cm.CmaEs.restart

    def spy(self, lam, mean, sigma):
        before = self.lr_state()
        orig(self, lam, mean, sigma)
        seen.append((before, self.lr_state()))
    monkeypatch.setattr(cm.CmaEs, "restart", spy)
    e = _experiment(f"lra-{strategy}", {"lr_adapt": "true", "restart_strategy": strategy, "random_state": 3})
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
    for before, after in seen:
        assert not _fresh(before, 4) and _fresh(after, 4)
    svc._exps[e.name].es.close()


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
    e = _experiment("lra-grpc", {"lr_adapt": "true", "popsize": 8, "random_state": 1})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=e))
    req = api.GetSuggestionsRequest(experiment=e, current_request_number=0)
    k, dup_gens = 0, 0
    rng = np.random.default_rng(0)
    loss = lambda a: (int(a["layers"]) - 4) ** 2 + (int(a["units"]) - 2) ** 2 + (np.log10(float(a["lr"])) + 2) ** 2 \
        + (float(a["dropout"]) - 0.2) ** 2 + 0.1 * rng.standard_normal()
    for gen in range(25):
        req.current_request_number = 8
        rep = stub.GetSuggestions(req)
        pts = [{x.name: x.value for x in pa.assignments} for pa in rep.parameter_assignments]
        assert len(pts) == 8
        assert all(a["layers"] in "123456" and a["units"] in "1234" and 0.001 <= float(a["lr"]) <= 0.1 for a in pts), pts
        dup_gens += len({(a["layers"], a["units"]) for a in pts}) < 8
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
    assert dup_gens > 0                      # integer parameters repeat, so the by-index matching was exercised
    assert svc._exps[e.name].es.lr_state()["eta_mean"] < 1.0
    svc._exps[e.name].es.close()
    ch.close()
    server.stop(0)
