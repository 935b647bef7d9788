"""GPU: skopt's GBRT surrogate (csrc/gbrt.cu) against the FP64 restatement oracle/gbrt_oracle.py, which tests/test_gbrt_oracle.py
holds to scikit-learn's chains.  Every stage's exported tree, the inits, μ, σ and the chain predictions are bit-identical to the
restatement; the acquisitions agree to 1e-12 and their first-index argmaxes are the restatement's."""
import numpy as np
import pytest

from kubeflow_b200.gbrt import GbrtEngine
from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Integer, Real
from oracle import gbrt_oracle as G

pytestmark = pytest.mark.gpu

KEYS = ("feature", "threshold", "left", "right", "value", "n_node_samples", "n_pos")


def _case(seed, N, D):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    X[:, ::2] = np.floor(X[:, ::2] * 8) / 7          # integer-like columns with many equal values
    y = np.sin(3 * X).sum(1) + 0.2 * rng.standard_normal(N)
    y[: N // 5] = np.round(y[: N // 5])              # tied y
    return X, y


def _assert_same_model(eng, chains):
    for c, ch in enumerate(chains):
        for s, t in enumerate(ch["trees"]):
            ex = eng.export(c, s)
            assert ex["init"] == ch["init"], f"chain {c}: init"
            for k in KEYS:
                assert np.array_equal(ex[k], t[k]), f"chain {c} stage {s}: {k} {ex[k]} != {t[k]}"


def _assert_same_predictions(eng, chains, Xc):
    mu, sd, q = G.predict(chains, Xc)
    dmu, dsd = eng.predict(Xc, return_std=True)
    assert np.array_equal(eng.predict(Xc, return_quantiles=True), q)
    assert np.array_equal(dmu, mu) and np.array_equal(dsd, sd)
    return mu, sd


@pytest.mark.parametrize("N", [1, 2, 3, 24, 250, 8192])
@pytest.mark.parametrize("D", [1, 4, 32])
def test_fit_equals_the_restatement_bit_for_bit(N, D):
    X, y = _case(N * 100 + D, N, D)
    eng = GbrtEngine()
    eng.tell(X, y)
    chains = G.fit(X, y)
    _assert_same_model(eng, chains)
    Xc = np.concatenate([np.random.default_rng(1).random((512, D)), X[:64]])
    _assert_same_predictions(eng, chains, Xc)
    if N == 8192:
        print(f"GBRT fit N={N} D={D}: {eng.last_timings()['fit_ms']:.2f} ms")
    eng.close()


def test_exact_binary_quantiles_and_constant_y():
    X, y = _case(7, 300, 3)
    eng = GbrtEngine(quantiles=(0.25, 0.5, 0.75))
    eng.tell(X, y)
    chains = G.fit(X, y, (0.25, 0.5, 0.75))
    _assert_same_model(eng, chains)
    _assert_same_predictions(eng, chains, X)
    eng.tell(X, np.full(300, 1.5))                                   # every node pure: one leaf per stage, σ = 0
    mu, sd = eng.predict(X, return_std=True)
    assert (mu == 1.5).all() and (sd == 0).all()
    b = eng.ask_multi(X, ["ei", "lcb", "pi"])
    assert [x.index for x in b] == [0, 0, 0] and b[0].value == 0.0 and b[2].value == 0.0
    eng.close()


def _thresholds(chains):
    out = []
    for ch in chains:
        for t in ch["trees"]:
            for f, th in zip(t["feature"], t["threshold"]):
                if f >= 0:
                    out.append((int(f), float(th)))
    return out


def test_decisions_at_a_million_candidates_with_every_threshold_neighbour():
    N, D, M = 2000, 8, 1 << 20
    X, y = _case(11, N, D)
    eng = GbrtEngine()
    eng.tell(X, y)
    chains = G.fit(X, y)
    rng = np.random.default_rng(12)
    Xc = rng.random((M, D)).astype(np.float32)
    r = 0
    for f, th in _thresholds(chains):          # candidates on the float32 neighbours of every threshold
        t32 = np.float32(th)
        for v in (np.nextafter(t32, np.float32(-1)), t32, np.nextafter(t32, np.float32(2))):
            Xc[r, f] = v
            r += 1
    mu, sd = _assert_same_predictions(eng, chains, Xc)
    y_opt = float(y.min())
    bests = eng.ask_multi(Xc, ["ei", "lcb", "pi"])
    for b, k in zip(bests, ("ei", "lcb", "pi")):
        ref = G.acquisition(k, mu, sd, y_opt)
        i = int(np.argmax(ref))
        assert b.index == i or abs(ref[b.index] - ref[i]) <= 1e-12 * max(1.0, abs(ref[i])), k
        assert abs(b.value - ref[b.index]) <= 1e-12 * max(1.0, abs(ref[b.index])), k
        assert b.mu == mu[b.index] and b.std == sd[b.index]
    print(f"GBRT sweep M={M} D={D}: {eng.last_timings()['sweep_ms']:.3f} ms")
    eng.close()


def test_crossing_quantiles_give_negative_sigma_zero_ei_and_lcb_as_is():
    for seed in range(50):                     # the first case whose quantiles cross at some candidate
        X, y = _case(seed, 40, 2)
        chains = G.fit(X, y)
        Xc = np.random.default_rng(seed).random((4096, 2))
        mu, sd, _ = G.predict(chains, Xc)
        if (sd < 0).any():
            break
    else:
        pytest.fail("no crossing case found")
    eng = GbrtEngine()
    eng.tell(X, y)
    _assert_same_predictions(eng, chains, Xc)
    (b_ei, b_lcb), dmu, dsd = eng.sweep(Xc, ["ei", "lcb"], return_arrays=True)
    ref_lcb = G.acquisition("lcb", mu, sd, float(y.min()))
    assert b_lcb.index == int(np.argmax(ref_lcb))
    assert sd[b_ei.index] > 0 or b_ei.value == 0.0
    eng.close()


def test_one_pass_hedge_equals_single_sweeps_and_a_sharded_sweep_the_whole():
    X, y = _case(21, 500, 5)
    eng = GbrtEngine()
    eng.tell(X, y)
    Xc = np.random.default_rng(22).random((100_000, 5))
    three = eng.ask_multi(Xc, ["ei", "lcb", "pi"])
    for b, k in zip(three, ("ei", "lcb", "pi")):
        eng.acq = k
        one = eng.ask(Xc)
        assert (one.index, one.value) == (b.index, b.value)
        parts = [eng.sweep(Xc[lo:hi], [k], global_offset=lo)[0] for lo, hi in ((0, 33_333), (33_333, 71_000), (71_000, 100_000))]
        best = max(parts, key=lambda p: (p.value, -p.index))
        assert (best.index, best.value) == (b.index, b.value)
    eng.close()


def test_optimizer_takes_an_engine_instance_and_refits_for_every_lie():
    eng = GbrtEngine()
    with pytest.raises(ValueError, match="GradientBoostingQuantileRegressor should run with acq_optimizer='sampling'"):
        Optimizer([Real(0.0, 1.0)], base_estimator=eng, acq_optimizer="lbfgs")
    space = [Real(-2.0, 2.0), Integer(0, 5), Real(0.0, 1.0)]
    opt = Optimizer(space, base_estimator=eng, n_initial_points=6, acq_func="gp_hedge", random_state=3, n_points=4096)
    rng = np.random.default_rng(4)
    pts = [[float(rng.uniform(-2, 2)), int(rng.integers(0, 6)), float(rng.random())] for _ in range(12)]
    opt.tell(pts, [p[0] ** 2 + 0.1 * p[1] + p[2] for p in pts])
    fits = []
    orig = eng.tell

    def spy(X, y):
        orig(X, y)
        fits.append((len(y), eng.last_fit))

    eng.tell = spy
    out = opt.ask(n_points=3)
    assert len(out) == 3 and fits == [(12, "fit"), (13, "fit"), (14, "fit")]
    Xt, yt = eng._hist
    chains = G.fit(Xt, yt)                              # the last lie's history
    _assert_same_model(eng, chains)
    opt.close()
    assert eng.N == 14                                 # the caller's engine stays open
    eng.close()
