"""GPU: ``multivariate-tpe``'s decisions against an exhaustive FP64 reference (tests/_mvtpe_ref.py, every candidate of every
point) at the shapes of record, for batches of points, at the score kernel's component-tile and the score and decision
kernels' candidate-block edges, through forced raises of the score kernel's running maximum, on infinite bounds, at the
integer offset table's limits and at the largest candidate count.

Every case asserts, over all candidates of every point, that the FP32 score lies within its bound of the FP64 score
(|s32 − s64| ≤ bound; the reference's own FP64 error is within _mvtpe_ref.tol, far below the bounds measured here), and that the engine's pick is np.argmax's, up to ties closer than two FP64 evaluations can separate (_mvtpe_ref.pick_ok)."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import mvtpe_oracle as O
from tests import _mvtpe_ref as R
from tests.test_gpu_mvtpe import SCORING_SPACE, engine, history, space_of

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
BUDGET = 1 << 25                  # candidates × components per reference chunk: 256 MiB per FP64 temporary


def check_point(space, models, out, p, what):
    """Bound and pick of point p of an ask with return_details; returns (median finite bound, max error / finite bound,
    distinct candidates within the FP64 tolerance of the maximum, infinite bounds)."""
    C = out["candidates"][p].T.contiguous()
    s64, T = R.score_tol(space, models, C, chunk=max(64, BUDGET // len(models["above"]["w"])))
    sc = out["scores"][p].double()
    err, e32 = (sc[:, 0] - s64).abs(), sc[:, 1]
    bad = ~(err <= e32)
    assert not bool(bad.any()), (f"{what} point {p}: |s32 - s64| > bound at {int(bad.sum())} of {C.shape[0]} candidates, "
                                 f"worst error / bound {float((err / e32).max()):.3g} at {int(torch.argmax(err / e32))}")
    fin = torch.isfinite(e32)
    ratio = float((err[fin] / e32[fin]).max()) if bool(fin.any()) else 0.0
    idx = int(out["index"][p])
    ok, msg, band = R.pick_ok(C, s64, T, idx)
    assert ok, f"{what} point {p}: {msg}"
    assert out["x"][p].tolist() == C[idx].tolist(), (what, p)
    return (float(e32[fin].median()) if bool(fin.any()) else math.nan), ratio, band, int((~fin).sum())


def report(what, out, res):
    """res: check_point's results, one per point."""
    s = out["survivors"]
    print(f"\n{what}: survivors per point min {s.min()} median {int(np.median(s))} max {s.max()}, "
          f"median bound {np.nanmedian([r[0] for r in res]):.2e}, max error / bound {max(r[1] for r in res):.3g}, "
          f"candidates within the FP64 tolerance of a maximum {max(r[2] for r in res)}, infinite bounds {sum(r[3] for r in res)}")


# ---- 1. shapes of record -----------------------------------------------------------------------------------------------------
RANGES = [(-1.0, 3.0), (0.0, 1e-3), (1e4, 1e4 + 1e-3), (-1e6, 1e6), (0.5, 0.5 + 1e-11)]
MIXED = [("float", 0.0, 1.0)] * 28 + [("int", 0, 19, 1), ("int", 0, (1 << 18) - 1, 1), ("cat", 3), ("cat", 10)]
RECORD = {
    "32 floats over five kinds of range, M=2^20": ([("float", *RANGES[d % len(RANGES)]) for d in range(32)], 1 << 20),
    "28 floats, integers of 20 and 2^18 levels, 2 categoricals, M=4096": (MIXED, 4096),
    "space_of(128), M=65536": (space_of(128), 65536),
}


@pytest.mark.parametrize("label", list(RECORD))
def test_shapes_of_record(label):
    """n = 8 192 trials, engine draws: DESIGN.md's cost table (32 floats at M = 2^20; the mixed space at M = 4 096) and the
    128-parameter mixed space of four float and eight discrete slabs."""
    space, M = RECORD[label]
    X, losses = history(space, 8192, seed=8192 + len(space))
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    out = t.ask(1, M, return_details=True)
    ms = t.last_timings()
    t.close()
    report(f"n=8192 {label}", out, [check_point(space, models, out, 0, label)])
    print("  engine phases (ms): " + ", ".join(f"{k} {v:.2f}" for k, v in ms.items()))


def test_largest_candidate_count():
    """n = 1 000, one float parameter, M = 2^24: the most candidates kbo_mvtpe_ask accepts."""
    space = [("float", -1.0, 3.0)]
    X, losses = history(space, 1000, seed=1000)
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    out = t.ask(1, 1 << 24, return_details=True)
    t.close()
    report("n=1000 D=1 M=2^24", out, [check_point(space, models, out, 0, "M=2^24")])


# ---- 2. batches of points ----------------------------------------------------------------------------------------------------
BATCH_SPACES = {"scoring": SCORING_SPACE, "space_of(40)": space_of(40)}


@pytest.mark.parametrize("M", [24, 4096, 65536])
@pytest.mark.parametrize("k", [2, 7])
@pytest.mark.parametrize("sname", list(BATCH_SPACES))
def test_batch_of_points_on_supplied_candidates(sname, k, M):
    """k points, each with its own candidates (the last point a copy of the first).  Every point is checked against the
    reference and equals the engine deciding that point alone: index, vector, survivors, candidates and scores."""
    space = BATCH_SPACES[sname]
    X, losses = history(space, 1000, seed=k * M + len(space))
    models = O.build_models(space, X, losses)
    r = np.random.default_rng(M + k)
    cands = np.stack([O.draw(space, models, M, r).T for _ in range(k)])
    cands[k - 1] = cands[0]
    assert not np.array_equal(cands[0], cands[1]) or k == 2
    C = torch.tensor(cands, device="cuda")
    t = engine(space, X, losses)
    out = t.ask(k, M, candidates=C, return_details=True)
    what = f"{sname} k={k} M={M}"
    res = [check_point(space, models, out, p, what) for p in range(k)]
    assert out["index"][k - 1] == out["index"][0] and np.array_equal(out["x"][k - 1], out["x"][0])
    for p in range(k):
        alone = t.ask(1, M, candidates=C[p:p + 1].contiguous(), return_details=True)
        assert alone["index"][0] == out["index"][p] and np.array_equal(alone["x"][0], out["x"][p]), (what, p)
        assert alone["survivors"][0] == out["survivors"][p], (what, p)
        assert torch.equal(alone["candidates"][0], out["candidates"][p]) and torch.equal(alone["scores"][0], out["scores"][p]), (what, p)
    t.close()
    report(what, out, res)


def test_batch_draws_differ_and_follow_the_below_model():
    """k = 4 points drawn by the engine, M = 2^18: the points' draws differ, each point's float marginals pass the KS test of
    test_sampler_distribution_joint_and_replay, and every point's decision matches the reference."""
    space = [("float", 0.0, 1.0), ("float", -1.0, 3.0), ("int", 3, 48, 5), ("cat", 4)]
    X, losses = history(space, 300, seed=5)
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses, seed=2024)
    M, k = 1 << 18, 4
    out = t.ask(k, M, return_details=True)
    t.close()
    C = out["candidates"].cpu().numpy()
    for p in range(k):
        for d in (0, 1):
            ks = stats.kstest(C[p, d], lambda x: O.marginal_cdf(space, models["below"], d, x))
            assert ks.statistic < 1.95 / np.sqrt(M), (p, d, ks)
        for p2 in range(p):
            assert not np.array_equal(C[p], C[p2]), (p, p2)
    report("drawn k=4 M=2^18", out, [check_point(space, models, out, p, "drawn k=4") for p in range(k)])


# ---- 3. component-tile and candidate-block edges -----------------------------------------------------------------------------
@pytest.mark.parametrize("n,ncomp", [(142, 127), (143, 128), (144, 129), (280, 255), (281, 256), (282, 257)])
def test_component_tile_and_candidate_block_edges(n, ncomp):
    """The above mixture has 127, 128, 129, 255, 256 or 257 components (the score kernel stages 128 at a time and pads the last
    tile), the below one 15 or 25; M runs over one candidate, partial and full score blocks of 64 and decision blocks of 256,
    and 2^20 + 1."""
    space = SCORING_SPACE
    X, losses = history(space, n, seed=n)
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    st = t.state()
    nb = 15 if n < 200 else 25
    assert len(st["above"]["w"]) - 1 == len(models["above"]["w"]) - 1 == ncomp
    assert len(st["below"]["w"]) - 1 == len(models["below"]["w"]) - 1 == st["n_below"] == nb
    for M in (1, 63, 64, 65, 255, 256, 257, (1 << 20) + 1):
        out = t.ask(1, M, return_details=True)
        report(f"n={n} ({ncomp} above components) M={M}", out, [check_point(space, models, out, 0, f"n={n} M={M}")])
    t.close()


# ---- 4. forced raises of the running maximum ---------------------------------------------------------------------------------
def _raises(space, g, x):
    """How often the score kernel raises its running maximum over group g's component tiles at the candidates x (K × D, a
    float-only space), by its rule (a thread's tile maximum above its running maximum + 64, log2), for each of a candidate
    row's 16 threads; the exponents in FP64 from the reference model.  Returns (K × 16)."""
    c, _, _ = R._group_terms(space, g)
    m = len(g["w"]) - 1
    z = (x[:, None, :] - g["mu"][None]) / g["sigma"]
    e = (c[:m] - 0.5 * (z * z).sum(-1)) * LOG2E
    nt = (m + 127) // 128
    e = np.pad(e, ((0, 0), (0, nt * 128 - m)), constant_values=-np.inf).reshape(len(x), nt, 128)
    cols = np.arange(16)[:, None] * 4 + np.array([0, 1, 2, 3, 64, 65, 66, 67])     # thread column tx's 8 components of a tile
    tmax = e[:, :, cols].max(-1)
    mref, n = np.full((len(x), 16), -np.inf), np.zeros((len(x), 16), dtype=int)
    for t in range(nt):
        up = tmax[:, t] > mref + 64
        mref, n = np.where(up, tmax[:, t], mref), n + up
    return n


@pytest.mark.parametrize("layout", ["closer", "away"])
def test_forced_raises_of_the_running_maximum(layout):
    """32 floats on [0, 1]; 25 below observations scattered, then 10 tiles of 128 identical above observations in told
    order.  Tile j sits at (d_j, …, d_j), with d_j such that its exponent at the origin lies 80·(9 − j) log2 units below the
    last tile's ("closer") or 80·j below the first's ("away", the control).  At 256 candidates within 0.01 of the origin the
    kernel's running maximum is then raised on every tile — ≥ 8 times, counted from the reference model — and the earlier
    tiles become far terms; in the control only once.  The other 3 840 candidates are draws from the below model."""
    D, J = 32, 10
    space = [("float", 0.0, 1.0)] * D
    sg = O.sigma(space[0], 128 * J, D)
    Q = 80.0 * (np.arange(J - 1, -1, -1) if layout == "closer" else np.arange(J))
    d = np.sqrt(Q / (D * LOG2E / (2 * sg * sg)))
    assert d.max() <= 1.0
    r = np.random.default_rng(4)
    X = np.concatenate([r.uniform(0.0, 1.0, (25, D)), np.repeat(d, 128)[:, None] * np.ones(D)])
    losses = np.concatenate([np.arange(25.0), 100.0 + r.random(128 * J)])
    models = O.build_models(space, X, losses)
    assert len(models["above"]["w"]) == 128 * J + 1 and models["above"]["sigma"][0] == sg
    near = r.uniform(0.0, 0.01, (256, D))
    nres = _raises(space, models["above"], near)
    if layout == "closer":
        assert nres.min() >= 8, nres.min()
    else:
        assert (nres == 1).all()
    cands = np.concatenate([near, O.draw(space, models, 4096 - 256, r)])
    cands = cands[r.permutation(len(cands))]
    t = engine(space, X, losses)
    out = t.ask(1, len(cands), candidates=torch.tensor(cands.T[None].copy(), device="cuda"), return_details=True)
    t.close()
    res = check_point(space, models, out, 0, layout)
    report(f"tiles moving {layout}: raises of the running maximum at the 256 chosen candidates {nres.min()}..{nres.max()}", out, [res])


# ---- 5. infinite bounds ------------------------------------------------------------------------------------------------------
def _lse_dt(space, g, x):
    """A lower bound on mv_lse_err's dt (the error of a near term's exponent, log2) for group g at the candidates x (K × D
    tensor, a float-only space), restated in FP64 from the reference model: the kernel's R = max(0, C_max + B − m + T + 1)
    with m, its running maximum, ≤ L = log2 of the group's density.  The kernel's bound is infinite where dt > ½."""
    u = 2.0 ** -24
    c, _, _ = R._group_terms(space, g)
    m = len(g["w"]) - 1
    c2 = c[:m] * LOG2E
    Df = len(space)
    XM = max((p[2] - p[1]) * math.sqrt(0.5 * LOG2E) / s for p, s in zip(space, g["sigma"]))
    L = R.log_density(space, g, x).cpu().numpy() * LOG2E
    Rr = np.maximum(0.0, c2.max() - L + 41.0)
    A = np.abs(c2).max() + Rr
    zeta = 2.02 * u * (XM * np.sqrt(Df * Rr) + Rr) + 2.05 * u * u * (Df * XM * XM + Rr)
    return 1.01 * (u * A + zeta + u * Df * A) + 1e-13 * A


def test_infinite_bounds_far_from_every_observation():
    """2 176 floats on [−1, 3], 1 000 observations within ±0.2 of the middle.  At a vector of range ends the prior dominates
    both densities, R ≈ 1.35 log2 units per parameter, and dt ≈ 1.01u·D·(|c|_max + R) grows as D²: by _lse_dt it is 0.15 at
    1 024 floats, 0.31 at 1 536, 0.54 at 2 048 and 0.61 at 2 176, the width used, so that it passes ½ with a margin
    (asserted).  256 such vectors mixed among 256 observed rows (dt ≈ 0.3: finite bounds) and 512 engine draws (dt up to
    about ½): every far vector has an infinite bound in the engine's output and survives into the FP64 pass, and the pick is
    still the FP64 argmax."""
    D, n = 2176, 1000
    space = [("float", -1.0, 3.0)] * D
    r = np.random.default_rng(D)
    X = 1.0 + r.uniform(-0.2, 0.2, (n, D))
    losses = r.random(n)
    models = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    drawn = t.ask(1, 512, return_details=True)["candidates"][0].T
    far = torch.tensor(np.where(r.random((256, D)) < 0.5, -1.0, 3.0), device="cuda")
    dt = np.maximum(_lse_dt(space, models["below"], far), _lse_dt(space, models["above"], far))
    assert dt.min() > 0.55, dt.min()
    kind = torch.tensor(r.permutation(np.repeat([0, 1, 2], [256, 256, 512])), device="cuda")    # far, observed, drawn
    cands = torch.empty(1024, D, dtype=torch.float64, device="cuda")
    cands[kind == 0], cands[kind == 1], cands[kind == 2] = far, torch.tensor(X[:256], device="cuda"), drawn
    out = t.ask(1, 1024, candidates=cands.T[None].contiguous(), return_details=True)
    t.close()
    inf = torch.isinf(out["scores"][0, :, 1])
    assert bool(inf[kind == 0].all()), int((~inf[kind == 0]).sum())
    assert out["survivors"][0] >= 256
    res = check_point(space, models, out, 0, "infinite bounds")
    report(f"D={D}: derived dt at the far vectors {dt.min():.3f}..{dt.max():.3f}; infinite bounds: far {int(inf[kind == 0].sum())} "
           f"of 256, observed {int(inf[kind == 1].sum())} of 256, drawn {int(inf[kind == 2].sum())} of 512", out, [res])


# ---- 6. the integer offset table's limits ------------------------------------------------------------------------------------
TABLE_SPACE = [("float", 0.0, 1.0), ("int", 0, 65535, 1), ("int", 0, 65536, 1), ("int", -7, -7 + 3 * 65535, 3), ("cat", 4)]


def test_integer_table_limits():
    """Two integers of exactly 2^16 levels, adjacent in the offset table (parameters 1 and 3, with another step and origin),
    and one of 2^16 + 1 levels between them (FP64 terms).  Observations sit on levels 0–2, candidates on every combination of
    levels {0, 1, levels − 1} — so the last entry of each table is read, where an offset one off would read the next table —
    then off the grid, half-way between grid points and outside the range, then draws.  The candidates as scored equal
    O.round_int's (both round half to even) before the decision is checked."""
    space = TABLE_SPACE
    ints = [1, 2, 3]
    r = np.random.default_rng(65536)
    n = 1000
    X = np.stack([r.uniform(0.0, 1.0, n)] + [O.bounds(space[d])[0] + r.integers(0, 3, n) * space[d][3] for d in ints]
                 + [r.integers(0, 4, n).astype(float)], axis=1)
    losses = r.random(n)
    models = O.build_models(space, X, losses)
    lv = [O.levels(space[d]) for d in ints]
    assert lv == [65536, 65537, 65536]
    rows = []
    for j in np.stack(np.meshgrid(*[[0, 1, L - 1] for L in lv], indexing="ij"), -1).reshape(-1, 3):
        rows.append([r.random()] + [O.bounds(space[d])[0] + jj * space[d][3] for d, jj in zip(ints, j)] + [float(r.integers(0, 4))])
    for f in (0.5, 1.5, 2.5, 0.3, -0.3, 65533.5, 65534.5, 65534.7, -0.4, -0.7, 65535.4, 65535.6, 12345.5):
        rows.append([r.random()] + [O.bounds(space[d])[0] + f * space[d][3] for d in ints] + [float(r.integers(0, 4))])
    cands = np.concatenate([np.asarray(rows), O.draw(space, models, 4096, r)])
    want = cands.copy()
    for d in ints:
        want[:, d] = O.round_int(space[d], cands[:, d])
    t = engine(space, X, losses)
    out = t.ask(1, len(cands), candidates=torch.tensor(cands.T[None].copy(), device="cuda"), return_details=True)
    t.close()
    assert np.array_equal(out["candidates"][0].cpu().numpy().T, want)
    for d, L in zip(ints, lv):
        assert (want[:, d] == O.bounds(space[d])[1]).sum() >= 9                          # level L - 1
    report("integers of 2^16, 2^16 + 1 and 2^16 levels", out, [check_point(space, models, out, 0, "integer table")])
