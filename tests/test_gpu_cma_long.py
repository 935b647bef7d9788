"""GPU: CMA-ES (kbo_cma_*) generation by generation over long runs, at the shapes Katib's `cmaes` uses, against the oracle.

Resynchronised parity: every generation the GPU's state (mean, σ, C, p_σ, p_c, generation count) is loaded into an
`oracle.CmaState`, `O.tell` is given the GPU's own steps Y and ‖z‖², and its result must match the GPU's next state.
Runs start where the service starts (mean 0.5, σ = 1/6, default popsize 4 + ⌊3 ln D⌋) and go on until C is numerically
singular (min eig < 1e3·ε·max eig), where the oracle itself stops meaning anything.  Every generation the eigendecomposition
is checked against `numpy.linalg.eigh` of the GPU's C, and d_j² must be λ_j itself, not a floor.

Tolerances are relative to each quantity's own scale (ε = 2.2e-16; ‖·‖₂ for C, ‖·‖ for vectors, |σ| for σ, never
max(1, ·)).  The rank-μ sum runs over λ samples, so C's carries √λ; p_σ and σ go through C^{-1/2}, so theirs carry
cond(C).  Each is 4× the worst value measured on an H100 80GB HBM3 (700 W power limit) over every run and ranking case
in this file, over two runs; the worst value is in brackets:
  mean       ‖Δm‖/‖m‖            ≤ 4·ε                 [0.995 ε]
  C          max|ΔC|/‖C‖₂         ≤ 3·ε·√λ              [0.68 ε·√λ, ranking at λ = 1024]
  p_c        ‖Δp_c‖/‖p_c‖         ≤ 370·ε               [93 ε, cigar D = 10]        
  p_σ        ‖Δp_σ‖/‖p_σ‖         ≤ 4000·ε·cond(C)      [965 ε·cond, D = 128, λ = 8192]
  σ          |Δσ|/σ               ≤ 210·ε·cond(C)       [52.5 ε·cond, D = 128, λ = 4096]
  BᵀB − I    max abs              ≤ 4e-13               [1.0004e-13: Jacobi stops at |g_a·g_b| ≤ 1e-13‖g_a‖‖g_b‖]
  C b − d² b max_j ‖·‖/‖C‖₂       ≤ 3500·ε              [864 ε, the same stopping rule]
  d² − eigh  max abs/‖C‖₂         ≤ 75·ε                [18.6 ε, cfg4 run at D = 128]
When the oracle's h_σ test lands within p_σ's tolerance of its threshold, either branch is accepted (no run needed it).
No run reached the singular horizon: every run stops at its generation count (400, 500, 1000, 600; 200 and 4 at D = 128).
On the parent commit, which floored every eigenvalue below 1e-8 and took d² as |λ|, the (2, 6) and
(4, 8) runs fail at the first generation whose min eig drops below 1e-8 (generations 89–120 and 128–243; eigenpair
residual 1e7–2e14 ε), and every ranking case fails on C (NaN ranked as +inf).
Jacobi sweeps per generation over the cfg4 run (200 generations, counting the final sweep that rotates nothing):
D = 128: 6 ×49, 7 ×138, 8 ×11, 9 ×1, 10 ×1; D = 127: 6 ×40, 7 ×149, 8 ×9, 9 ×1, 10 ×1.  The cap is 30.
"""
import json

import numpy as np
import pytest
import torch

from oracle import cma_oracle as O

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps

TOL_MEAN, TOL_C, TOL_PC, TOL_PS, TOL_SIGMA = 4.0, 3.0, 370.0, 4000.0, 210.0
TOL_ORTH, TOL_PAIR, TOL_EIG = 4e-13, 3500.0, 75.0


def _record(name, **kv):
    print(f"\nMEASURED {name} " + json.dumps(kv))


def _es(D, lam, seed, mean=0.5, sigma=1.0 / 6.0):
    from kubeflow_b200.cmaes import CmaEs
    return CmaEs(np.full(D, mean), sigma, popsize=lam, seed=seed)


def _eigen_errors(st):
    """(‖BᵀB − I‖max, max_j ‖C b_j − d_j² b_j‖/‖C‖₂ in ε, max|sort(d²) − eigh|/‖C‖₂ in ε, eigh's eigenvalues)"""
    C, B, d = st["C"], st["B"], st["d"]
    ev = np.linalg.eigvalsh(C)
    n2 = max(abs(ev[0]), abs(ev[-1]))
    orth = np.abs(B.T @ B - np.eye(len(d))).max()
    pair = np.linalg.norm(C @ B - B * d * d, axis=0).max() / n2 / EPS
    eig = np.abs(np.sort(d * d) - ev).max() / n2 / EPS
    return orth, pair, eig, ev


def _load(st, lam):
    ref = O.CmaState(st["mean"], st["sigma"], lam)
    ref.C, ref.p_sigma, ref.pc, ref.g = st["C"].copy(), st["p_sigma"].copy(), st["pc"].copy(), st["generation"]
    return ref


def _errors(ref, got, cond):
    """errors in the units of the tolerances: ε, ε·√λ for C, ε·cond(C) for p_σ and σ"""
    rel = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b) / EPS if np.linalg.norm(b) > 0 else np.linalg.norm(a) / EPS
    lam = ref.p.popsize
    return dict(mean=rel(got["mean"], ref.mean), C=np.abs(got["C"] - ref.C).max() / np.linalg.norm(ref.C, 2) / EPS / np.sqrt(lam),
                pc=rel(got["pc"], ref.pc), ps=rel(got["p_sigma"], ref.p_sigma) / cond,
                sigma=abs(got["sigma"] - ref.sigma) / ref.sigma / EPS / cond)


LIMITS = dict(mean=TOL_MEAN, C=TOL_C, pc=TOL_PC, ps=TOL_PS, sigma=TOL_SIGMA)


def resync_run(D, lam, name, gens, seed=0):
    """Drive a CmaEs from the service's start on objective `name`; check each generation against the oracle resynchronised
    to the GPU's state.  Returns (generation where the run stopped, worst normalised errors, generations that took the other h_σ branch)."""
    f, _, _ = O.objective(name, D, seed)
    es = _es(D, lam, seed)
    r = np.random.default_rng(seed + 1)
    worst = dict(mean=0.0, C=0.0, pc=0.0, ps=0.0, sigma=0.0, orth=0.0, pair=0.0, eig=0.0)
    prev, stop, hflips = None, gens, 0
    for g in range(gens + 1):
        z = r.standard_normal((lam, D))
        X = es.ask(torch.tensor(z, device="cuda")).cpu().numpy()
        st = es.state(with_Y=True)
        assert st["generation"] == g
        orth, pair, eig, ev = _eigen_errors(st)
        if prev is not None:
            ref, alt, cond = prev
            err = _errors(ref, st, cond)
            if alt is not None:                         # h_σ within rounding of its threshold: either branch
                err2 = _errors(alt, st, cond)
                if max(err2[k] / LIMITS[k] for k in LIMITS) < max(err[k] / LIMITS[k] for k in LIMITS):
                    err, hflips = err2, hflips + 1
            for k in LIMITS:
                worst[k] = max(worst[k], err[k])
                assert err[k] <= LIMITS[k], f"{name} D={D} lam={lam} generation {g}: {k} error {err[k]:.3g} > {LIMITS[k]} " \
                                            f"(cond(C) {cond:.3g}, min eig {ev[0]:.3g}, sigma {st['sigma']:.3g})"
        if ev[0] < 1e3 * EPS * ev[-1]:
            stop = g
            break
        worst["orth"], worst["pair"], worst["eig"] = max(worst["orth"], orth), max(worst["pair"], pair), max(worst["eig"], eig)
        where = f"{name} D={D} lam={lam} generation {g} (min eig {ev[0]:.3g}, max {ev[-1]:.3g})"
        assert orth <= TOL_ORTH, f"{where}: |B'B - I| = {orth:.3g}"
        assert pair <= TOL_PAIR, f"{where}: eigenpair residual {pair:.3g} eps"
        assert eig <= TOL_EIG, f"{where}: d^2 vs eigh {eig:.3g} eps (d^2 min {np.min(st['d'] ** 2):.3g})"
        if g == gens:
            break
        fx = f(X)
        es.tell(fx)
        cond = ev[-1] / ev[0]
        zn2 = (z * z).sum(1)
        ref = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2)
        p = ref.p
        h_left = np.linalg.norm(ref.p_sigma) / np.sqrt(1 - (1 - p.c_sigma) ** (2 * (st["generation"] + 1)))
        thr = (1.4 + 2 / (D + 1)) * p.chi_n
        alt = None
        if abs(h_left - thr) <= TOL_PS * EPS * cond * h_left:
            h = 1.0 if h_left < thr else 0.0
            alt = O.tell(_load(st, lam), st["Y"], fx, znorm2=zn2, h_sigma=1.0 - h)
        prev = (ref, alt, cond)
    es.close()
    return stop, worst, hflips


LONG = [(2, 6, 400), (4, 8, 500), (10, 10, 1000), (32, 14, 600)]


@pytest.mark.parametrize("name", O.OBJECTIVES)
@pytest.mark.parametrize("D,lam,gens", LONG, ids=[f"D{d}-lam{l}" for d, l, _ in LONG])
def test_long_run_resynchronised_parity(D, lam, gens, name):
    assert lam == 4 + int(3 * np.log(D))                  # the service's default population
    stop, worst, hflips = resync_run(D, lam, name, gens)
    _record(f"resync {name} D={D} lam={lam}", stopped_at=stop, hflips=hflips, **worst)


@pytest.mark.parametrize("D,lam,gens,name", [(128, 4096, 200, "ellipsoid1e6"), (128, 8192, 4, "sphere")])
def test_cfg4_scale_resynchronised_parity(D, lam, gens, name):
    stop, worst, hflips = resync_run(D, lam, name, gens)
    _record(f"resync {name} D={D} lam={lam}", stopped_at=stop, hflips=hflips, **worst)


@pytest.mark.parametrize("D", [128, 127])
def test_jacobi_over_cfg4_run(D):
    """The run bench.py times (Rastrigin from mean 3, σ 2, λ = 4096), one generation per call so each generation's sweep
    count is seen; the eigendecomposition is checked after every generation."""
    es = _es(D, 4096, 7, mean=3.0, sigma=2.0)
    sweeps, worst = [], [0.0, 0.0, 0.0]
    for g in range(200):
        out = es.run_synthetic("rastrigin", 1)
        sweeps.append(int(out["jacobi_sweeps"]))
        st = es.state()
        orth, pair, eig, ev = _eigen_errors(st)
        worst = [max(worst[0], orth), max(worst[1], pair), max(worst[2], eig)]
        assert ev[0] > 1e3 * EPS * ev[-1]
        assert orth <= TOL_ORTH and pair <= TOL_PAIR and eig <= TOL_EIG, (g, orth, pair, eig)
    es.close()
    hist = {int(k): int(v) for k, v in zip(*np.unique(sweeps, return_counts=True))}
    _record(f"jacobi D={D}", sweeps_hist=hist, sweeps_last50=sorted(set(sweeps[-50:])), orth=worst[0], pair=worst[1], eig=worst[2])
    assert max(sweeps) < 30, hist                              # the cap (30) is never reached


RANK_LAMBDAS = [4, 5, 6, 255, 256, 257, 1024, 1025, 4097, 8192]


def _rank_fitness(lam, seed):
    r = np.random.default_rng(seed)
    f = np.round(r.standard_normal(lam) * 3.0) / 2.0           # plateaus, as integer parameters give: many ties
    k = max(lam // 16, 1)
    for v in (np.nan, np.inf, -np.inf, 0.0, -0.0, np.copysign(np.nan, -1.0)):
        f[r.choice(lam, k, replace=False)] = v
    special = [np.nan, np.inf, -0.0, -np.inf, 0.0, np.copysign(np.nan, -1.0)]
    f[:min(lam, 6)] = special[:min(lam, 6)]                    # a NaN ahead of a +inf, a -0 ahead of a +0
    return f


@pytest.mark.parametrize("lam", RANK_LAMBDAS)
def test_ranking_follows_numpy_order(lam):
    """NaN after +inf, -0 == +0, ties by sample index: the update must be the oracle's (lexsort) one."""
    D = 3
    es = _es(D, lam, lam)
    r = np.random.default_rng(lam)
    z = r.standard_normal((lam, D))
    es.ask(torch.tensor(z, device="cuda"))
    st = es.state(with_Y=True)
    worst = dict(mean=0.0, C=0.0, pc=0.0, ps=0.0, sigma=0.0)
    for gen in range(2):
        f = _rank_fitness(lam, 100 * lam + gen)
        es.tell(f)
        ref = O.tell(_load(st, lam), st["Y"], f, znorm2=(z * z).sum(1))
        z = r.standard_normal((lam, D))
        es.ask(torch.tensor(z, device="cuda"))
        got = es.state(with_Y=True)
        err = _errors(ref, got, 1.0)
        for k in worst:
            worst[k] = max(worst[k], err[k])
            assert err[k] <= LIMITS[k], (gen, k, err)
        st = got
    es.close()
    _record(f"rank lam={lam}", **worst)


@pytest.mark.parametrize("kind", ["sphere", "rastrigin"])
@pytest.mark.parametrize("D,lam,G", [(24, 48, 100), (128, 4096, 10)])
def test_run_synthetic_is_ask_fitness_tell(D, lam, G, kind):
    """kbo_cma_run_synthetic (bench.py's cfg4 path) performs exactly the generations ask() / host fitness / tell() do."""
    a, b = _es(D, lam, 11, mean=3.0, sigma=2.0), _es(D, lam, 11, mean=3.0, sigma=2.0)
    a.run_synthetic(kind, G)
    fn = O.sphere if kind == "sphere" else O.rastrigin
    for g in range(G):
        X = b.ask().cpu().numpy()
        f = fn(X)
        # the device's sum order and cospi may differ from the host's by a few ulps per term: the order must not hinge on it
        bound = 8 * EPS * D * (X * X + 20.0 + 20.0 * np.pi * np.abs(X)).sum(1)
        o = np.argsort(f)
        gaps = np.diff(f[o])
        assert (gaps > bound[o][1:] + bound[o][:-1]).all(), f"generation {g}: two fitness values too close to rank reliably"
        b.tell(f)
    sa, sb = a.state(), b.state()
    for k in ("mean", "sigma", "C", "B", "d", "p_sigma", "pc", "generation"):
        assert np.array_equal(sa[k], sb[k]), k
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------ built-in sampler
def _philox_normals(n, seed, gen):
    """NumPy restatement of cma_normal_kernel: Philox4x32-10 on counter (pair, generation), key seed; Box–Muller in FP64."""
    M = np.uint64(0xFFFFFFFF)
    p = np.arange((n + 1) // 2, dtype=np.uint64)
    c0, c1 = p & M, p >> np.uint64(32)
    c2, c3 = np.full_like(p, np.uint64(gen) & M), np.full_like(p, np.uint64(gen) >> np.uint64(32))
    k0, k1 = np.uint64(seed) & M, np.uint64(seed) >> np.uint64(32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    u1 = (((c0 << np.uint64(21)) ^ (c1 >> np.uint64(11))).astype(np.float64) + 1.0) * (1.0 / 9007199254740993.0)
    u2 = ((c2 << np.uint64(21)) ^ (c3 >> np.uint64(11))).astype(np.float64) * (1.0 / 9007199254740992.0)
    rad = np.sqrt(-2.0 * np.log(u1))
    z = np.empty(2 * len(p))
    z[0::2], z[1::2] = rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)
    return z[:n]


def _first_draw(D, lam, seed):
    es = _es(D, lam, seed, mean=0.0, sigma=1.0)             # B = I, d = 1: x = z exactly
    X = es.ask().cpu().numpy().copy()
    return es, X


@pytest.mark.parametrize("D,lam,seed", [(3, 5, 0), (1, 7, 3), (37, 9, 1 << 40), (128, 8192, 123)])
def test_sampler_is_philox_box_muller(D, lam, seed):
    """Odd λ·D (the last Box–Muller pair half used) included; generation 1 checked through the updated B and d."""
    es, X = _first_draw(D, lam, seed)
    np.testing.assert_allclose(X.ravel(), _philox_normals(D * lam, seed, 0), rtol=0, atol=1e-13)
    if (D * lam) % 2:
        es2, X2 = _first_draw(D, lam + 1, seed)            # same stream, one more sample
        assert np.array_equal(X2.ravel()[:D * lam], X.ravel())
        es2.close()
    es.tell(np.arange(lam, dtype=np.float64))
    es.ask()
    st = es.state(with_Y=True)
    z1 = (st["Y"] @ st["B"]) / st["d"]
    np.testing.assert_allclose(z1.ravel(), _philox_normals(D * lam, seed, 1), rtol=0, atol=1e-10)
    es.close()


def test_sampler_statistics_seeds_and_generations():
    from scipy import stats
    D, lam = 128, 8192
    es, X = _first_draw(D, lam, 2024)
    z = X.ravel()
    n = z.size
    ks = stats.kstest(z, "norm")
    m, v = z.mean(), z.var()
    sk, ku = stats.skew(z), stats.kurtosis(z)
    _record("sampler", n=n, ks_p=ks.pvalue, mean=m, var=v, skew=sk, kurt=ku)
    assert ks.pvalue > 1e-3
    assert abs(m) < 5 / np.sqrt(n) and abs(v - 1) < 5 * np.sqrt(2 / n)
    assert abs(sk) < 5 * np.sqrt(6 / n) and abs(ku) < 5 * np.sqrt(24 / n)
    # a second handle with the same seed draws the same generation bit for bit
    es2, X2 = _first_draw(D, lam, 2024)
    assert np.array_equal(X, X2)
    es2.close()
    # seeds that differ only in their high 32 bits give different, uncorrelated streams
    es3, X3 = _first_draw(D, lam, 2024 + (1 << 32))
    assert not np.array_equal(X, X3) and abs(np.corrcoef(z, X3.ravel())[0, 1]) < 5 / np.sqrt(n)
    es3.close()
    # consecutive generations are uncorrelated (generation 1 read back through B and d)
    es.tell(np.zeros(lam))
    es.ask()
    st = es.state(with_Y=True)
    z1 = ((st["Y"] @ st["B"]) / st["d"]).ravel()
    assert abs(np.corrcoef(z, z1)[0, 1]) < 5 / np.sqrt(n)
    assert stats.kstest(z1, "norm").pvalue > 1e-3
    es.close()
