"""GPU: ``tpe``'s decisions against an exhaustive FP64 reference (tests/_tpe_ref.py, every candidate of every (point, parameter))
at the shapes of record, for batches of points, at the component-chunk and score-tile edges, under non-default gamma and
prior_weight, on forced FP64 decisions and past the 65 536-level table; and the service's batches over gRPC.

Every continuous case asserts, over all candidates, that the FP32 score lies within its bound of the FP64 score
(|s32 − s64| ≤ e32; the reference's own FP64 error, ≤ 1e-11, is far below the smallest bound, 1e-9), and every (point,
parameter) that the engine's pick is np.argmax's, up to ties closer than two FP64 evaluations can separate (_tpe_ref.tol)."""
import grpc
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import tpe_oracle as O
from tests import _tpe_ref as R
from tests.test_gpu_tpe import _experiment, _multiset, _objective, _units, engine, history

pytestmark = pytest.mark.gpu

MIXED = [("uniform", -1.0, 3.0), ("quniform", 0.0, 20.0, 1.0), ("choice", 64), ("uniform", 1e4, 1e4 + 1e-3),
         ("quniform", 3.0, 48.0, 5.0), ("choice", 4)]


def check_point(space, models, out, p, what):
    """Bound and pick of every parameter of point p of an ask with return_details; returns (median bound, max error / bound)
    over its continuous parameters and the most keys any parameter had within tolerance of its maximum (1: the pick was
    checked exactly)."""
    C = out["candidates"][p]
    med, ratio, band = [], 0.0, 1
    for d, (sp, m) in enumerate(zip(space, models)):
        x = C[d]
        s64 = R.score(m, x)
        idx = int(out["index"][p, d])
        if sp[0] == "uniform":
            sc = out["scores"][p, d].double()
            err, e32 = (sc[:, 0] - s64).abs(), sc[:, 1]
            bad = ~(err <= e32)
            assert not bool(bad.any()), (f"{what} point {p} param {d} {sp}: |s32 - s64| > bound at {int(bad.sum())} of {x.shape[0]} "
                                         f"candidates, worst error / bound {float((err / e32).max()):.3g}")
            med.append(float(e32.median()))
            ratio = max(ratio, float((err / e32).max()))
        ok, msg, nk = R.pick_ok(m, x, s64, idx)
        assert ok, f"{what} point {p} param {d} {sp}: {msg}"
        band = max(band, nk)
        v = float(x[idx])
        if sp[0] == "quniform":
            v = float(O.quantize(v, sp[3]))
        assert out["x"][p, d] == v, (what, p, d)
    return (float(np.median(med)) if med else float("nan")), ratio, band


def report(what, out, res):
    """res: check_point's results, one per point."""
    s = out["survivors"]
    print(f"\n{what}: survivors per (point, parameter) min {s.min()} median {int(np.median(s))} max {s.max()}, "
          f"median bound {np.nanmedian([r[0] for r in res]):.2e}, max error / bound {max(r[1] for r in res):.3g}, "
          f"keys within the FP64 tolerance of a maximum {max(r[2] for r in res)}")


# ---- 1. shapes of record -----------------------------------------------------------------------------------------------------
RANGES = [(-1.0, 3.0), (0.0, 1e-3), (1e4, 1e4 + 1e-3), (-1e6, 1e6), (0.5, 0.5 + 1e-11)]   # the last: sigma's 1e-12 floor binds


def test_shapes_of_record():
    """n = 8 192, D = 32 uniform parameters over five kinds of range, M = 2^20 engine draws.  history()'s ties put many sigma at
    the ps/100 floor (r' = 100)."""
    space = [("uniform", *RANGES[d % len(RANGES)]) for d in range(32)]
    X, losses = history(space, 8192, seed=8192)
    models, _ = O.build_models(space, X, losses)
    for m, sp in zip(models, space):
        assert np.sum(m["above"]["sigma"] == (sp[2] - sp[1]) / 100) > 4096, sp
    t = engine(space, X, losses)
    out = t.ask(1, 1 << 20, return_details=True)
    t.close()
    report("n=8192 D=32 M=2^20", out, [check_point(space, models, out, 0, "n=8192 D=32 M=2^20")])


def test_largest_candidate_count():
    """n = 1 000, one parameter, M = 2^24: the service's n_EI_candidates limit."""
    space = [("uniform", -1.0, 3.0)]
    X, losses = history(space, 1000, seed=1000)
    models, _ = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    out = t.ask(1, 1 << 24, return_details=True)
    t.close()
    report("n=1000 D=1 M=2^24", out, [check_point(space, models, out, 0, "n=1000 M=2^24")])


# ---- 2. batches of points ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [24, 4096, 65536])
@pytest.mark.parametrize("k", [2, 7])
def test_batch_of_points_on_supplied_candidates(k, M):
    """k points over the mixed space, each with its own candidates (the last point a copy of the first).  Every (point,
    parameter) is checked against the reference and equals the engine deciding that point alone, scores included."""
    space = MIXED
    X, losses = history(space, 1000, seed=k * M)
    models, _ = O.build_models(space, X, losses)
    r = np.random.default_rng(M + k)
    cands = np.stack([np.stack([O.draw(m, M, r) for m in models]) for _ in range(k)])
    cands[k - 1] = cands[0]
    assert not np.array_equal(cands[0], cands[1]) or k == 2
    C = torch.tensor(cands, device="cuda")
    t = engine(space, X, losses)
    out = t.ask(k, M, candidates=C, return_details=True)
    what = f"k={k} M={M}"
    res = [check_point(space, models, out, p, what) for p in range(k)]
    assert np.array_equal(out["index"][k - 1], out["index"][0]) and np.array_equal(out["x"][k - 1], out["x"][0])
    for p in range(k):
        alone = t.ask(1, M, candidates=C[p:p + 1].contiguous(), return_details=True)
        assert np.array_equal(alone["index"][0], out["index"][p]) and np.array_equal(alone["x"][0], out["x"][p]), (what, p)
        assert np.array_equal(alone["survivors"][0], out["survivors"][p]), (what, p)
        cont = [d for d, sp in enumerate(space) if sp[0] == "uniform"]
        assert torch.equal(alone["scores"][0, cont], out["scores"][p, cont]), (what, p)
    t.close()
    report(what, out, res)


def test_batch_draws_differ_and_follow_the_below_model():
    """k = 4 points drawn by the engine, M = 2^18: the points' draws differ, each point's draws pass the KS test of
    test_sampler_distribution_bounds_and_determinism, and every point's decisions match the reference."""
    space = [("uniform", -1.0, 3.0), ("quniform", 3.0, 48.0, 5.0), ("choice", 4)]
    X, losses = history(space, 300, seed=5)
    t = engine(space, X, losses, seed=2024)
    M, k = 1 << 18, 4
    out = t.ask(k, M, return_details=True)
    st = t.state()
    t.close()
    C = out["candidates"].cpu().numpy()
    for p in range(k):
        for d, (lo, hi) in ((0, (-1.0, 3.0)), (1, (3.0, 48.0))):
            assert (C[p, d] >= lo).all() and (C[p, d] < hi).all()
            b = st[d]["below"]
            ks = stats.kstest(C[p, d], lambda x: O.truncated_mixture_cdf(x, b["w"], b["mu"], b["sigma"], lo, hi))
            assert ks.statistic < 1.95 / np.sqrt(M), (p, d, ks)
            for p2 in range(p):
                assert not np.array_equal(C[p, d], C[p2, d]), (p, p2, d)
        counts = np.bincount(C[p, 2].astype(int), minlength=4) / M
        assert np.abs(counts - st[2]["below"]["p"]).max() < 5e-3      # 5 standard deviations of a proportion at M = 2^18
    models, _ = O.build_models(space, X, losses)
    res = [check_point(space, models, out, p, "drawn k=4") for p in range(k)]
    report("drawn k=4 M=2^18", out, res)


# ---- 3. component-chunk and score-tile edges ---------------------------------------------------------------------------------
@pytest.mark.parametrize("n,ncomp", [(1032, 1024), (1033, 1025), (2059, 2048), (2060, 2049)])
def test_chunk_and_tile_edges(n, ncomp):
    """The above mixture at gamma = 0.25 has exactly 1 024, 1 025, 2 048 or 2 049 components (the FP32 pass stages 1 024 at a
    time); M runs over one candidate, partial and full 1 024-candidate tiles and 2^20 + 1."""
    space = [("uniform", -1.0, 3.0), ("uniform", 0.5, 0.5 + 1e-11)]
    X, losses = history(space, n, seed=n)
    models, _ = O.build_models(space, X, losses)
    t = engine(space, X, losses)
    assert [len(s["above"]["w"]) for s in t.state()] == [ncomp, ncomp] == [len(m["above"]["w"]) for m in models]
    for M in (1, 1023, 1024, 1025, (1 << 20) + 1):
        out = t.ask(1, M, return_details=True)
        report(f"n={n} ({ncomp} components) M={M}", out, [check_point(space, models, out, 0, f"n={n} M={M}")])
    t.close()


# ---- 4. forced FP64 decisions ------------------------------------------------------------------------------------------------
def _ref_maximiser(model, lo, hi, dev="cuda"):
    """The reference score's best interior local maximiser on [lo, hi) (the global one may sit on an end of the range, with no
    room for candidates on both sides): the best strict local maximum of a 2^20 grid, then four zooms of 4 097 points onto
    the neighbourhood of the best so far."""
    x = torch.linspace(lo, hi, (1 << 20) + 1, dtype=torch.float64, device=dev)[:-1]
    s = R.score(model, x)
    peak = torch.nonzero((s[1:-1] > s[:-2]) & (s[1:-1] > s[2:])).flatten() + 1
    i = int(peak[torch.argmax(s[peak])])
    for _ in range(4):
        x = torch.linspace(float(x[i - 1]), float(x[i + 1]), 4097, dtype=torch.float64, device=dev)
        i = min(max(int(torch.argmax(R.score(model, x))), 1), 4095)
    return float(x[i])


def test_forced_fp64_decision():
    """4 096 distinct candidates within ±1e-6·range of a reference maximiser, the maximiser itself at index 2 731 and a copy
    of it at index 4 096: the FP32 scores cannot order them, so every candidate survives into the FP64 pass, which must pick
    the maximiser's first copy.  The others keep at least 5e-7·range from it, so that the maximiser beats them by more than
    the two FP64 evaluations' tolerance (asserted)."""
    lo, hi = -1.0, 3.0
    space = [("uniform", lo, hi)]
    X, losses = history(space, 8192, seed=77)
    models, _ = O.build_models(space, X, losses)
    m = models[0]
    xs = _ref_maximiser(m, lo, hi)
    rg = 1e-6 * (hi - lo)
    r = np.random.default_rng(3)
    off = np.linspace(0.5 * rg, 0.999 * rg, 2048)                      # below rg, so that xs ± off rounds to within rg
    x = np.concatenate([xs + off, xs - off[:2047]])
    x = x[r.permutation(len(x))]
    x = np.concatenate([x[:2731], [xs], x[2731:], [xs]])
    assert len(np.unique(x[:-1])) == 4096 and (np.abs(x - xs) <= rg).all() and x[0] != xs
    C = torch.tensor(x, device="cuda")
    s64 = R.score(m, C)
    assert x[int(torch.argmax(s64))] == xs           # either copy: torch's reductions may round equal rows differently
    T = R.tol(m, C)
    assert bool((s64[2731] - s64[:2731] > T[2731] + T[:2731]).all()) and bool((s64[2731] - s64[2732:-1] > T[2731] + T[2732:-1]).all())
    t = engine(space, X, losses)
    out = t.ask(1, len(x), candidates=C[None, None], return_details=True)
    t.close()
    assert out["survivors"][0, 0] == len(x)
    assert out["index"][0, 0] == 2731 and out["x"][0, 0] == xs
    report("forced FP64 decision", out, [check_point(space, models, out, 0, "forced")])


# ---- 5. gamma and prior_weight -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [30, 8192])
@pytest.mark.parametrize("prior_weight", [1e-3, 50.0])
@pytest.mark.parametrize("gamma", [0.05, 0.9])
def test_settings(gamma, prior_weight, n):
    space = MIXED
    X, losses = history(space, n, seed=n + int(gamma * 100))
    t = engine(space, X, losses, gamma=gamma, prior_weight=prior_weight)
    got = t.state()
    ref, nb = O.build_models(space, X, losses, gamma=gamma, prior_weight=prior_weight)
    for d, (g, m) in enumerate(zip(got, ref)):
        assert g["n_below"] == nb
        for grp in ("below", "above"):
            if m["kind"] == "choice":
                np.testing.assert_allclose(g[grp]["p"], m[grp], rtol=1e-13, atol=0)
                continue
            a, b = g[grp], m[grp]
            assert len(a["w"]) == len(b["w"]), (d, grp)
            np.testing.assert_allclose(_multiset(a["mu"], a["sigma"], a["w"]), _multiset(b["mu"], b["sigma"], b["w"]), rtol=1e-13, atol=0,
                                       err_msg=f"param {d} {grp}")
            assert abs(a["p_accept"] - b["p_accept"]) <= 1e-13 * b["p_accept"]
    out = t.ask(1, 4096, return_details=True)
    t.close()
    what = f"gamma={gamma} prior_weight={prior_weight} n={n}"
    report(what, out, [check_point(space, ref, out, 0, what)])


# ---- 6. discrete parameters past the level table -----------------------------------------------------------------------------
def _level_candidates(p, best, r):
    """Every level, its neighbours ±0.3 and the half-levels j + ½ (rounding half to even), lo and the largest double below
    hi, shuffled; then three more candidates on the best level at later indices."""
    if p[0] == "choice":
        c = r.permutation(p[1]).astype(np.float64)
        return np.concatenate([c, [best, best, best]])
    lo, hi, q = p[1], p[2], p[3]
    j = np.arange(lo, hi + q / 2, q)
    c = np.concatenate([j, (j + 0.5 * q)[:-1], j[1:] - 0.3 * q, (j + 0.3 * q)[:-1], [lo, np.nextafter(hi, lo)]])
    c = c[r.permutation(len(c))]
    return np.concatenate([c, [best, best + 0.2 * q if best < hi else best - 0.2 * q, best - 0.2 * q if best > lo else best]])


@pytest.mark.parametrize("p,table", [(("quniform", 0.0, 65535.0, 1.0), True), (("quniform", 0.0, 65536.0, 1.0), False),
                                     (("quniform", 0.0, float(1 << 18), 1.0), False), (("choice", 65536), True),
                                     (("choice", 65537), False)], ids=["q65536", "q65537", "q262145", "c65536", "c65537"])
def test_discrete_past_the_level_table(p, table):
    """Up to 65 536 levels each level present is scored once (survivors = levels); past that every candidate is (survivors =
    M).  Either way the pick is the best level's first occurrence.  Quantized scores are compared under _tpe_ref.tol (at
    2^18 levels Φ(ub) − Φ(lb) cancels to about 1e-10 relative, and CUDA's erf and torch's differ by ulps); choices exactly."""
    space = [p]
    L = p[1] if p[0] == "choice" else int(round((p[2] - p[1]) / p[3])) + 1
    X, losses = history(space, 1000, seed=L)
    models, _ = O.build_models(space, X, losses)
    m = models[0]
    lv = torch.arange(L, dtype=torch.float64, device="cuda") * (1.0 if p[0] == "choice" else p[3]) + (0.0 if p[0] == "choice" else p[1])
    best = float(lv[int(torch.argmax(R.score(m, lv)))])
    x = _level_candidates(p, best, np.random.default_rng(L))
    C = torch.tensor(x, device="cuda")
    assert torch.equal(torch.unique(R.key(m, C)), lv)                   # every level present
    t = engine(space, X, losses)
    out = t.ask(1, len(x), candidates=C[None, None], return_details=True)
    t.close()
    assert out["survivors"][0, 0] == (L if table else len(x))
    idx = int(out["index"][0, 0])
    assert idx < len(x) - 3                                               # the appended copies come after the first occurrence
    s = R.score(m, C)
    ok, msg, band = R.pick_ok(m, C, s, idx)
    assert ok, f"{p}: {msg}"
    v = float(x[idx]) if p[0] == "choice" else float(O.quantize(x[idx], p[3]))
    assert out["x"][0, 0] == v
    print(f"\n{p}: M={len(x)} survivors {out['survivors'][0, 0]}, pick {idx} (level {v}), levels within tolerance of the best: {band}")


# ---- the service's batches over gRPC -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tpe_batch_stub():
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    from kubeflow_b200.suggestion.tpe_service import TpeService
    svc = TpeService()
    server, port = serve(DispatchService([svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


@pytest.mark.parametrize("k", [3, 5])
def test_service_batches_match_oracle(tpe_batch_stub, k):
    """Rounds of k points (n_EI_candidates 64, random_state fixed).  A replica engine with the same seed, history and ask count
    regenerates the k × D × 64 candidates of each model-based round; every point of every reply is the oracle's choice over
    its own candidates."""
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.internal import HyperParameterSearchSpace
    from kubeflow_b200.suggestion.tpe_service import tpe_space
    from kubeflow_b200.tpe import Tpe
    stub, svc = tpe_batch_stub
    name = f"svc-batch-{k}"
    settings = {"random_state": 7, "n_EI_candidates": 64}
    exp = _experiment(name, settings)
    space = tpe_space(HyperParameterSearchSpace.convert(exp))
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=k)
    replica = Tpe(space, seed=7)
    rows, losses, model_rounds = [], [], 0
    for i in range(16):
        rep = stub.GetSuggestions(req)
        pts = [{x.name: x.value for x in pa.assignments} for pa in rep.parameter_assignments]
        assert len(pts) == k
        if len(rows) >= 20:                                   # n_startup_jobs: model-based from here on
            model_rounds += 1
            replica.tell(np.asarray(rows[replica.n:]), np.asarray(losses[replica.n:]))
            out = replica.ask(k, 64, return_details=True)
            models, _ = O.build_models(space, np.asarray(rows), np.asarray(losses))
            cands = out["candidates"].cpu().numpy()
            for p, a in enumerate(pts):
                vals, _ = O.choose(models, cands[p])
                assert _units(a) == vals.tolist() == out["x"][p].tolist(), (i, p)
            assert len({a["x"] for a in pts}) == k
        else:
            assert svc._exps[name].engine is None
        for j, a in enumerate(pts):
            tr = req.trials.add()
            tr.name = f"{name}-t{i}-{j}"
            tr.spec.objective.objective_metric_name = "acc"
            for kk, v in a.items():
                x = tr.spec.parameter_assignments.assignments.add()
                x.name, x.value = kk, v
            tr.status.condition = api.SUCCEEDED
            mm = tr.status.observation.metrics.add()
            mm.name, mm.value = "acc", repr(_objective(a))
            rows.append(_units(a))
            losses.append(-_objective(a))
    replica.close()
    assert model_rounds >= 8
