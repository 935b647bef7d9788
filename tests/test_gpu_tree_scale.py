"""GPU: the tree surrogates (csrc/forest.cu, csrc/gbrt.cu) on every fit and sweep variant their sizes select, against the FP64
restatements oracle/forest_oracle.py and oracle/gbrt_oracle.py.  Trees, μ, σ and chain predictions are bit for bit; picks follow
the rules of tests/test_gpu_forest.py and tests/test_gpu_gbrt.py.

The forest sweep stages each tree in shared memory when the largest one fits there beside the kernel's own static shared memory,
and walks it in global memory otherwise; the CTAs per SM follow from the same sizes.  The GBRT sweep stages a 256-row candidate
tile beside its model while both fit in 113 KiB.  The forest fit runs its trees in batches whose column scratch stays within 2 GiB.
Each case below asserts which of these variants it reaches."""
import ctypes as C
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest
import torch

from kubeflow_b200 import _lib as L
from kubeflow_b200.forest import ForestEngine
from kubeflow_b200.gbrt import GbrtEngine
from oracle import forest_oracle as F
from oracle import gbrt_oracle as G
from tests._forest_ref import assert_same_tree, dyadic_case

pytestmark = pytest.mark.gpu

# H100: a block may opt in to 227 KiB of shared memory, static and dynamic together; an SM has 228 KiB, and the system reserves
# 1 KiB of it per resident block.  Every forest_sweep_kernel instance has 768 static bytes (TreeArgmax's partials), pinned on the
# CPU by tests/test_sass_forest.py::test_sweep_kernels_static_shared_memory_is_the_size_the_staging_band_assumes.
OPTIN, SM_SHARED, RESERVED = 232448, 233472, 1024
SWEEP_STATIC = 768
FOREST_MAX_N, FOREST_MAX_D = 65536, 1024


def tree_bytes(tree):
    """Packed size of one tree in the sweep: 16-byte leaf records, then 8-byte nodes padded to an even count."""
    n = len(tree["left"])
    return 16 * int((tree["left"] < 0).sum()) + 8 * (n + n % 2)


def sweep_variant(max_bytes):
    """(staged, CTAs per SM that shared memory allows) of the forest sweep for its largest packed tree, or (False, None): walked
    in global memory."""
    if max_bytes + SWEEP_STATIC > OPTIN:
        return False, None
    return True, SM_SHARED // (max_bytes + SWEEP_STATIC + RESERVED)


# With a tree of L single-sample leaves (2L − 1 nodes, 32·L bytes) the largest tree staged is L = 7240, and 2 CTAs fit up to
# L = 3592: both band edges, each with a case on either side and at the old literals' edges (113 KiB = 32·3616, 227 KiB = 32·7264).
STAGE_MAX_LEAVES = (OPTIN - SWEEP_STATIC) // 32
OCC2_MAX_LEAVES = (SM_SHARED // 2 - SWEEP_STATIC - RESERVED) // 32
assert (STAGE_MAX_LEAVES, OCC2_MAX_LEAVES) == (7240, 3592)


def _launch(eng):
    st = (C.c_int32 * 6)()
    eng.check(eng.lib.kbo_debug_forest_sweep(eng._h, eng._o, st))
    return dict(zip(("staged", "cpt", "occ", "nblocks", "static", "optin"), list(st)))


def _assert_variant(eng, max_bytes, cpt):
    """The last sweep's launch is the variant its largest tree selects.  Registers allow every staged instance (at most 114 per
    thread) 2 CTAs per SM, so where shared memory allows at most 2 it alone decides."""
    got = _launch(eng)
    assert (got["static"], got["optin"]) == (SWEEP_STATIC, OPTIN), got
    staged, occ = sweep_variant(max_bytes)
    assert bool(got["staged"]) == staged and got["cpt"] == cpt, (max_bytes, got)
    if staged:
        assert got["occ"] == occ if occ <= 2 else 2 <= got["occ"] <= occ, (max_bytes, got)
    return "global" if not staged else f"staged, {got['occ']} CTA/SM"


def _candidates(rng, trees, M, D):
    """Uniform rows, with a share of them exactly on each split's fp32 neighbours (RD and RU of the FP64 threshold), integer-grid
    and one-hot values in columns 0 and 1 (as tests/test_gpu_forest.py)."""
    Xc = rng.random((M, D)).astype(np.float32)
    if D > 1:
        Xc[: M // 8, 0] = rng.integers(0, 9, M // 8) / 8.0
        Xc[: M // 8, 1] = rng.integers(0, 2, M // 8)
    fs, vs = [], []
    for tr in trees:
        k = np.flatnonzero(tr["left"] >= 0)
        th = tr["threshold"][k]
        rd = th.astype(np.float32)
        rd = np.where(rd.astype(np.float64) > th, np.nextafter(rd, np.float32(-np.inf)), rd)
        ru = np.nextafter(rd, np.float32(np.inf))
        fs += [tr["feature"][k], tr["feature"][k]]
        vs += [rd, ru]
    f, v = np.concatenate(fs), np.concatenate(vs)
    Xc[rng.integers(M // 8, M, len(f)), f] = v
    return Xc


def _predict(trees, Xc):
    """F.predict, over row blocks in worker processes at a million candidates: the restatement walks 2^20 rows through 100 trees
    in about 100 s on one core.  Rows are independent, so the blocks concatenate to F.predict(trees, Xc) exactly."""
    if len(Xc) <= 65536:
        return F.predict(trees, Xc)
    blocks = np.array_split(Xc, min(os.cpu_count() or 1, 32))
    with ProcessPoolExecutor(len(blocks), mp_context=multiprocessing.get_context("fork")) as ex:
        out = list(ex.map(F.predict, [trees] * len(blocks), blocks))
    return np.concatenate([o[0] for o in out]), np.concatenate([o[1] for o in out])


def _check_pick(b, v, mu, sd):
    """tests/test_gpu_forest.py's rule on precomputed acquisition values v: the pick is a maximum to 1e-13, no earlier row has
    its (μ, σ), and it reports the row's μ and σ."""
    top = v.max()
    assert v[b.index] >= top - 1e-13 * max(abs(top), 1e-300), f"picked {v[b.index]!r}, max {top!r}"
    same = np.flatnonzero((mu[: b.index] == mu[b.index]) & (sd[: b.index] == sd[b.index]))
    assert len(same) == 0, f"index {b.index} has an earlier twin {same[:3]}"
    assert b.mu == mu[b.index] and b.std == sd[b.index]


ACQS = ("ei", "lcb", "pi")


def _check_sweep(eng, Xc, mu, sd, vals, goff=0):
    """One sweep per acquisition with μ and σ on every row, then the three-way hedge at global_offset goff."""
    Xd = torch.from_numpy(Xc).cuda()
    for acq in ACQS:
        (b,), mu_d, sd_d = eng.sweep(Xd, [acq], return_arrays=True)
        assert np.array_equal(mu_d.cpu().numpy(), mu), f"{acq}: mu"
        assert np.array_equal(sd_d.cpu().numpy(), sd), f"{acq}: sigma"
        _check_pick(b, vals[acq], mu, sd)
    for acq, b in zip(ACQS, eng.sweep(Xd, list(ACQS), global_offset=goff)):
        assert b.index >= goff
        b.index -= goff
        _check_pick(b, vals[acq], mu, sd)


def _acq_values(eng, mu, sd):
    return {a: F.acquisition(a, mu, sd, eng.y_opt, eng.xi, eng.kappa) for a in ACQS}


def _et_draws(seed, t):
    return lambda k, f, a, b: F.et_threshold(F.et_uniform(seed, t, k, f), a, b)


def _node_minmax(tree, X):
    """min / max of every feature over each node's samples (ET: every sample is in the root)."""
    n, D = len(tree["left"]), X.shape[1]
    mn, mx = np.full((n, D), np.inf, np.float32), np.full((n, D), -np.inf, np.float32)
    members = {0: np.arange(len(X))}
    for k in range(n):
        r = members.pop(k)
        if tree["left"][k] < 0:
            continue
        mn[k], mx[k] = X[r].min(axis=0), X[r].max(axis=0)
        go = X[r, tree["feature"][k]].astype(np.float64) <= tree["threshold"][k]
        members[tree["left"][k]], members[tree["right"][k]] = r[go], r[~go]
    return mn, mx


def _check_et_tree(eng, X, y, seed, t):
    """ET tree t and the thresholds drawn at each of its nodes against the Philox restatement."""
    ex = eng.export(t, with_draws=True)
    assert_same_tree(ex, F.build_tree(X, y, None, kind="ET", draws=_et_draws(seed, t)), rtol=0, where=f"ET tree {t}")
    mn, mx = _node_minmax(ex, X)
    n, D = mn.shape
    inner = ex["left"] >= 0
    k, f = np.meshgrid(np.arange(n), np.arange(D), indexing="ij")
    const = mx <= (mn + F.FEATURE_THRESHOLD)
    want = np.where(inner[:, None] & ~const, F.et_threshold(F.et_uniform(seed, t, k, f), mn, mx), np.nan)
    assert np.array_equal(ex["draws"], want, equal_nan=True), f"ET tree {t}: drawn thresholds"
    kk = np.flatnonzero(inner)
    assert np.array_equal(ex["threshold"][kk], ex["draws"][kk, ex["feature"][kk]])


# ---- (a) the staging band, with exact leaf counts --------------------------------------------------------------------------
@pytest.mark.parametrize("N", [3592, 3593, 3616, 3617, 7240, 7241, 7264, 7265])
def test_forest_sweep_on_each_side_of_the_staging_and_occupancy_edges(N):
    """Tree 0 of an RF with min_samples_leaf = 1 on all-ones counts, N distinct x and N distinct y grows exactly N single-sample
    leaves, so its packed size is 32·N; trees 1-3 draw bootstrap counts and come out smaller."""
    T, seed = 4, 7
    rng = np.random.default_rng(N)
    X = np.empty((N, 2), np.float32)
    X[:, 0] = rng.permutation(N) / np.float32(N)                  # distinct values 1/N apart, far above 1e-7
    X[:, 1] = rng.random(N)
    y = (rng.permutation(N) - N // 2) / 4096.0                    # distinct multiples of 2^-12
    counts = F.bootstrap_counts(N, T, seed)
    counts[0] = 1
    eng = ForestEngine(kind="RF", n_trees=T, min_samples_leaf=1, seed=seed)
    eng.tell(X, y, counts=counts)
    trees = [eng.export(t) for t in range(T)]
    assert len(trees[0]["left"]) == 2 * N - 1 and int((trees[0]["left"] < 0).sum()) == N
    assert max(tree_bytes(t) for t in trees) == tree_bytes(trees[0]) == 32 * N
    for t in (0, 1):
        assert_same_tree(trees[t], F.build_tree(X, y, counts[t], min_samples_leaf=1, kind="RF"), rtol=0, where=f"tree {t}")
    Xc = _candidates(rng, trees, 1 << 20, 2)
    mu, sd = _predict(trees, Xc)
    vals = _acq_values(eng, mu, sd)
    variants = []
    for M, cpt in ((65536, 1), (1 << 20, 4)):
        _check_sweep(eng, Xc[:M], mu[:M], sd[:M], {a: v[:M] for a, v in vals.items()}, goff=12345)
        variants.append(_assert_variant(eng, 32 * N, cpt))
    mu_p, sd_p = eng.predict(Xc[:4096])
    assert np.array_equal(mu_p, mu[:4096]) and np.array_equal(sd_p, sd[:4096])
    variants.append(_assert_variant(eng, 32 * N, 1))
    print(f"band N={N}: {32 * N} B, sweep {set(variants)}")
    eng.close()


# ---- (b) natural large histories, and the limits ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind,N,variant", [("ET", 16384, "staged, 1 CTA/SM"), ("RF", 16384, "staged, 2 CTA/SM"),
                                            ("ET", 65536, "global"), ("RF", 65536, "global")])
def test_forest_at_large_histories_against_the_restatement(kind, N, variant):
    D, T, seed = 8, 100, 99
    rng = np.random.default_rng(N + D)
    X, y = dyadic_case(rng, N, D, grid=True)
    eng = ForestEngine(kind=kind, n_trees=T, seed=seed)
    eng.tell(X, y)
    fit_ms = eng.last_timings()["fit_ms"]
    trees = [eng.export(t) for t in range(T)]
    max_bytes = max(tree_bytes(t) for t in trees)
    counts = F.bootstrap_counts(N, T, seed) if kind == "RF" else None
    for t in (0, 99):
        if kind == "RF":
            assert np.array_equal(trees[t]["counts"], counts[t])
            assert_same_tree(trees[t], F.build_tree(X, y, counts[t], kind="RF"), rtol=0, where=f"RF tree {t}")
        else:
            _check_et_tree(eng, X, y, seed, t)
    Xc = _candidates(rng, trees, 65536, D)
    mu, sd = _predict(trees, Xc)
    _check_sweep(eng, Xc, mu, sd, _acq_values(eng, mu, sd))
    assert _assert_variant(eng, max_bytes, 1) == variant
    print(f"{kind} N={N} D={D} T={T}: largest tree {max_bytes} B ({variant}), fit {fit_ms:.1f} ms, "
          f"sweep M=65536 {eng.last_timings()['sweep_ms']:.2f} ms")
    if N == 16384:       # the limits are refused and the fitted forest stays usable
        with pytest.raises(L.KboInvalidArgument):
            eng.tell(np.zeros((FOREST_MAX_N + 1, D)), np.zeros(FOREST_MAX_N + 1))
        with pytest.raises(L.KboInvalidArgument):
            eng.tell(np.zeros((10, FOREST_MAX_D + 1)), np.arange(10.0))
        mu_p, sd_p = eng.predict(Xc[:1000])
        assert np.array_equal(mu_p, mu[:1000]) and np.array_equal(sd_p, sd[:1000])
        eng.tell(X[:500], y[:500])
        mu_p, _ = eng.predict(Xc[:1000])
        assert np.array_equal(mu_p, F.predict([eng.export(t) for t in range(T)], Xc[:1000])[0])
    eng.close()


# ---- (c) the record shape, swept ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["RF", "ET"])
def test_forest_at_the_record_shape_over_a_million_candidates(kind):
    N, D, T, seed, M = 8192, 32, 100, 4242, 1 << 20
    rng = np.random.default_rng(31)
    X, y = dyadic_case(rng, N, D, grid=True)
    eng = ForestEngine(kind=kind, n_trees=T, seed=seed)
    eng.tell(X, y)
    trees = [eng.export(t) for t in range(T)]
    if kind == "ET":
        for t in (0, 50, 99):
            _check_et_tree(eng, X, y, seed, t)
    Xc = _candidates(rng, trees, M, D)
    mu, sd = _predict(trees, Xc)
    _check_sweep(eng, Xc, mu, sd, _acq_values(eng, mu, sd), goff=7 << 30)
    variant = _assert_variant(eng, max(tree_bytes(t) for t in trees), 4)
    print(f"{kind} record shape: fit {eng.last_timings()['fit_ms']:.1f} ms, sweep M={M} {eng.last_timings()['sweep_ms']:.2f} ms "
          f"({variant})")
    eng.close()


# ---- (d) the batched fit and wide features -----------------------------------------------------------------------------------
def test_rf_fit_in_two_batches_at_512_features():
    N, D, T, seed = 8192, 512, 100, 5
    cap = 2 * max(1, N // 3) + 1
    batch = min(T, (2 << 30) // (2 * 4 * N * D + N + 8 * cap))     # trees per launch: column scratch within 2 GiB
    assert batch == 63
    X, y = dyadic_case(np.random.default_rng(512), N, D, grid=True)
    eng = ForestEngine(kind="RF", n_trees=T, seed=seed)
    eng.tell(X, y)
    print(f"RF fit N={N} D={D} T={T} (batches of {batch}): {eng.last_timings()['fit_ms']:.1f} ms")
    counts = F.bootstrap_counts(N, T, seed)
    for t in (0, batch - 1, batch, T - 1):
        ex = eng.export(t)
        assert np.array_equal(ex["counts"], counts[t])
        assert_same_tree(ex, F.build_tree(X, y, counts[t], kind="RF"), rtol=0, where=f"tree {t}")
    eng.close()


@pytest.mark.parametrize("kind", ["RF", "ET"])
def test_forest_splits_and_sweeps_features_past_511(kind):
    """D = FOREST_MAX_D with y driven by columns 1000 and 1023: splits on features whose index fills the packed node's 10-bit
    feature field."""
    N, D, T, seed = 400, FOREST_MAX_D, 10, 8
    rng = np.random.default_rng(1024)
    X = rng.random((N, D)).astype(np.float32)
    y = np.sin(4.0 * X[:, 1000]) + X[:, 1023] ** 2 + 0.05 * rng.standard_normal(N)
    y = np.round(y * 4096.0) / 4096.0
    eng = ForestEngine(kind=kind, n_trees=T, seed=seed)
    eng.tell(X, y)
    trees = [eng.export(t) for t in range(T)]
    feats = np.concatenate([t["feature"][t["left"] >= 0] for t in trees])
    assert (feats >= 512).any() and (feats >= 1000).any()
    if kind == "RF":
        assert_same_tree(trees[0], F.build_tree(X, y, F.bootstrap_counts(N, T, seed)[0], kind="RF"), rtol=0, where="tree 0")
    else:
        _check_et_tree(eng, X, y, seed, 0)
    Xc = _candidates(rng, trees, 65536, D)
    mu, sd = _predict(trees, Xc)
    _check_sweep(eng, Xc, mu, sd, _acq_values(eng, mu, sd))
    _assert_variant(eng, max(tree_bytes(t) for t in trees), 1)
    eng.close()


# ---- (e) GBRT across its staging edge and limits -----------------------------------------------------------------------------
GBRT_TILE_LIMIT = 113 * 1024


def gbrt_staged(S, D):
    """The GBRT sweep stages a 256-row candidate tile (pitch D | 1) beside its model (3 chains × S stages × 15 heap slots of a
    double and a uint2) while both fit in 113 KiB."""
    return 3 * S * 15 * 16 + 256 * (D | 1) * 4 <= GBRT_TILE_LIMIT


def test_gbrt_cases_straddle_the_staging_predicate():
    assert gbrt_staged(30, 91) and not gbrt_staged(30, 92)
    assert gbrt_staged(128, 23) and not gbrt_staged(128, 24)


def _gbrt_case(rng, N, D, col):
    X = rng.random((N, D))
    X[:, ::2] = np.floor(X[:, ::2] * 8) / 7                      # integer-like columns with many equal values
    if col is None:
        y = np.sin(3 * X).sum(1) + 0.2 * rng.standard_normal(N)
    else:
        y = np.sin(6 * X[:, col]) + 0.2 * rng.standard_normal(N)
    y[: N // 5] = np.round(y[: N // 5])                          # tied y
    return X, y


@pytest.mark.parametrize("S,D,N,col", [(30, 91, 2000, None), (30, 92, 2000, None), (128, 23, 2000, None), (128, 24, 2000, None),
                                       (1, 4, 2000, None), (10, 1024, 300, 1023), (30, 4, 65536, None)])
def test_gbrt_against_the_restatement_across_its_staging_edge_and_limits(S, D, N, col):
    rng = np.random.default_rng(S * 10000 + D + N)
    X, y = _gbrt_case(rng, N, D, col)
    eng = GbrtEngine(n_estimators=S)
    eng.tell(X, y)
    fit_ms = eng.last_timings()["fit_ms"]
    chains = G.fit(X, y, n_stages=S)
    for c, ch in enumerate(chains):
        for s, t in enumerate(ch["trees"]):
            ex = eng.export(c, s)
            assert ex["init"] == ch["init"], f"chain {c}: init"
            for k in ("feature", "threshold", "left", "right", "value", "n_node_samples", "n_pos"):
                assert np.array_equal(ex[k], t[k]), f"chain {c} stage {s}: {k}"
    if col is not None:
        assert any((t["feature"] == col).any() for ch in chains for t in ch["trees"])
    Xc = rng.random((65536, D)).astype(np.float32)
    r = 0
    for ch in chains:                                           # the float32 neighbours of every threshold
        for t in ch["trees"]:
            for f, th in zip(t["feature"], t["threshold"]):
                if f < 0:
                    continue
                t32 = np.float32(th)
                for v in (np.nextafter(t32, np.float32(-1)), t32, np.nextafter(t32, np.float32(2))):
                    Xc[r % len(Xc), f] = v
                    r += 1
    Xc[-64:] = X[:64]
    mu, sd, q = G.predict(chains, Xc)
    assert np.array_equal(eng.predict(Xc, return_quantiles=True), q)
    dmu, dsd = eng.predict(Xc, return_std=True)
    assert np.array_equal(dmu, mu) and np.array_equal(dsd, sd)
    bests, mu_d, sd_d = eng.sweep(Xc, list(ACQS), return_arrays=True)
    assert np.array_equal(mu_d.cpu().numpy(), mu) and np.array_equal(sd_d.cpu().numpy(), sd)
    y_opt = float(y.min())
    for b, k in zip(bests, ACQS):
        ref = G.acquisition(k, mu, sd, y_opt)
        i = int(np.argmax(ref))
        assert b.index == i or abs(ref[b.index] - ref[i]) <= 1e-12 * max(1.0, abs(ref[i])), k
        assert abs(b.value - ref[b.index]) <= 1e-12 * max(1.0, abs(ref[b.index])), k
        assert b.mu == mu[b.index] and b.std == sd[b.index]
    print(f"GBRT S={S} D={D} N={N} ({'staged' if gbrt_staged(S, D) else 'unstaged'} tile): fit {fit_ms:.2f} ms, "
          f"sweep M={len(Xc)} {eng.last_timings()['sweep_ms']:.3f} ms")
    eng.close()
