"""GPU: the ENAS controller (kbo_enas_*) against the FP64 oracle — teacher-forced training parity over 50 steps, sampling
parity on imposed uniforms, the distribution of 2^16 draws, bit-for-bit determinism, and the ``enas`` service over gRPC."""
import json

import grpc
import numpy as np
import pytest
from scipy import stats as ss

from oracle import enas_oracle as O

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1), (8, 64, 78), (12, 64, 6), (24, 128, 1024), (64, 128, 4096)]
NONE_VARIANTS = [("temperature",), ("tanh_const",), ("temperature", "tanh_const"), ("entropy_weight", "skip_weight")]


def _controller(L, H, n_ops, st, seed=1):
    from kubeflow_b200.enas import EnasController
    return EnasController(L, H, n_ops, settings=st, seed=seed)


def _random_arcs(rng, T, L, n_ops):
    out = np.zeros((T, L * (L + 1) // 2), np.int32)
    for t in range(T):
        for l in range(L):
            pos = l * (l + 1) // 2
            out[t, pos] = rng.integers(n_ops)
            out[t, pos + 1:pos + 1 + l] = rng.random(l) < 0.4
    return out


def _parity(L, H, n_ops, st, R=0.8, T=50, p_tol=1e-6):
    ctl = _controller(L, H, n_ops, st)
    s0 = ctl.state()
    arcs = _random_arcs(np.random.default_rng(L * 1000 + n_ops), T, L, n_ops)
    gpu = ctl.train(R, T, arcs=arcs)
    s1 = ctl.state()
    ref = O.new_state(s0["params"])
    scale = max(1.0, abs(R))
    worst = {n: 0.0 for n in ("nll", "ent", "kl", "baseline", "loss")}
    rows = []
    for t in range(T):
        o = O.train_step(ref, L, st, R, arc=arcs[t])
        rows.append(o)
        for i, n in enumerate(("nll", "ent", "kl")):         # kl relative to its terms' magnitude: they cancel near the target
            worst[n] = max(worst[n], abs(gpu[t, i] - o[n]) / max(o["kl_abs"] if n == "kl" else abs(o[n]), 1e-30))
        worst["baseline"] = max(worst["baseline"], abs(gpu[t, 4] - o["baseline"]) / scale)
        worst["loss"] = max(worst["loss"], abs(gpu[t, 3] - o["loss"]) / (scale + abs(o["loss"])))
        assert gpu[t, 5] == pytest.approx(o["skip_rate"], abs=1e-6)
    perr = {n: float(np.abs(s1["params"][n] - ref["params"][n]).max()) for n in O.PARAM_NAMES}
    print(f"parity L={L} H={H} n_ops={n_ops} lr={st['learning_rate']}: worst relative stats {worst}, parameter errors {perr}")
    for n in ("nll", "ent", "kl", "baseline"):
        assert worst[n] <= 1e-5, (n, worst[n])
    # the loss carries the cancellation in r - baseline (absolute bound) and, while the baseline is far from r, it is
    # nll·(r - b) (up to ~1500 at L = 64), which inherits nll's own 1e-5 relative bound: the second term
    assert worst["loss"] <= 1e-5, worst["loss"]
    for n in O.PARAM_NAMES:
        assert perr[n] <= p_tol, (n, perr[n])
    assert s1["step"] == T and s1["draws"] == T and abs(s1["baseline"] - ref["baseline"]) <= 1e-5 * scale
    ctl.close()


@pytest.mark.parametrize("L,H,n_ops", SHAPES)
def test_teacher_forced_parity(L, H, n_ops):
    _parity(L, H, n_ops, O.settings())


@pytest.mark.parametrize("L,H,n_ops", [(8, 64, 78), (12, 64, 6)])
def test_teacher_forced_parity_at_high_learning_rate(L, H, n_ops):
    """lr = 0.05, step by step from the GPU's own state.  Run free for 50 steps, the FP32 and FP64 trajectories separate at
    this rate: with β1 = 0, Adam maps a gradient difference dg to a step difference of up to lr·sqrt(1 - β2)/ε̂·dg ≈ 1.6·dg, so
    each step's rounding is amplified by the next.  Each step here starts the oracle from the exported state (parameters,
    moments, baseline, Adam step) and holds that one step to the 1e-5 parameter bound and the stats bounds."""
    st = O.settings(learning_rate=0.05)
    R, T = 0.8, 50
    ctl = _controller(L, H, n_ops, st)
    arcs = _random_arcs(np.random.default_rng(L * 1000 + n_ops), T, L, n_ops)
    worst_p = 0.0
    for t in range(T):
        s = ctl.state()
        ref = dict(params={n: a.astype(np.float64) for n, a in s["params"].items()}, m={n: a.astype(np.float64) for n, a in s["m"].items()},
                   v={n: a.astype(np.float64) for n, a in s["v"].items()}, baseline=float(s["baseline"]), step=s["step"])
        g = ctl.train(R, 1, arcs=arcs[t:t + 1])[0]
        o = O.train_step(ref, L, st, R, arc=arcs[t])
        for i, n in enumerate(("nll", "ent", "kl")):
            assert abs(g[i] - o[n]) <= 1e-5 * (o["kl_abs"] if n == "kl" else abs(o[n])) + 1e-30, (t, n, g[i], o[n])
        assert abs(g[4] - o["baseline"]) <= 1e-5 * max(1.0, R)
        assert abs(g[3] - o["loss"]) <= 1e-5 * (max(1.0, R) + abs(o["loss"]))
        s1 = ctl.state()
        for n in O.PARAM_NAMES:
            worst_p = max(worst_p, float(np.abs(s1["params"][n] - ref["params"][n]).max()))
    print(f"high-lr parity L={L} H={H} n_ops={n_ops}: largest one-step parameter error {worst_p:.2e}")
    assert worst_p <= 1e-5 and ctl.state()["step"] == T
    ctl.close()


@pytest.mark.parametrize("none", NONE_VARIANTS)
def test_teacher_forced_parity_with_none_settings(none):
    _parity(8, 64, 78, O.settings(**{k: None for k in none}))


def test_sampling_parity_on_imposed_uniforms():
    L, H, n_ops, k = 8, 64, 78, 1024
    st = O.settings()
    ctl = _controller(L, H, n_ops, st, seed=3)
    P = {n: a * 8 for n, a in ctl.state()["params"].items()}       # a crafted controller: far from uniform probabilities
    ctl.set_params(P)
    U = np.random.default_rng(5).random((k, L * (L + 1) // 2)).astype(np.float32)
    arcs, opp, skp = ctl.sample(k, uniforms=U, return_probs=True)
    P64 = {n: a.astype(np.float64) for n, a in ctl.state()["params"].items()}
    near = 0
    for a in range(k):
        fw = O.forward(P64, L, st, arc=arcs[a])             # the oracle's probabilities along the GPU's own arc
        probs = []
        for l in range(L):
            probs.append(fw["op_p"][l])
            probs += [np.array([1 - p, p]) for p in fw["skip_p"][l * (l - 1) // 2:l * (l + 1) // 2]]
        for d, p in enumerate(probs):
            want = O.draw(p, float(U[a, d]))
            if want != arcs[a, d]:
                c = np.concatenate([[0.0], np.cumsum(p)])
                b = max(want, int(arcs[a, d]))
                assert abs(int(arcs[a, d]) - want) == 1 and abs(float(U[a, d]) - c[b]) <= 1e-5, (a, d, want, arcs[a, d])
                near += 1
        np.testing.assert_allclose(opp[a], np.array(fw["op_p"]), rtol=0, atol=1e-5)
        np.testing.assert_allclose(skp[a], fw["skip_p"], rtol=0, atol=1e-5)
    print(f"sampling parity: {k} arcs, {near} decisions differed within 1e-5 of a CDF boundary")
    ctl.close()


def test_distribution_of_draws():
    L, H, n_ops = 4, 16, 7
    st = O.settings()
    ctl = _controller(L, H, n_ops, st, seed=11)
    ctl.set_params({n: a * 10 for n, a in ctl.state()["params"].items()})
    arcs, opp, skp = [], [], []
    for _ in range(64):                                     # 2^16 arcs
        a, o, s = ctl.sample(1024, return_probs=True)
        arcs.append(a), opp.append(o), skp.append(s)
    arcs, opp, skp = np.concatenate(arcs), np.concatenate(opp), np.concatenate(skp)
    P64 = {n: a.astype(np.float64) for n, a in ctl.state()["params"].items()}
    for a in range(0, len(arcs), 4096):                     # the probabilities the test weighs with are the oracle's
        fw = O.forward(P64, L, st, arc=arcs[a])
        np.testing.assert_allclose(opp[a], np.array(fw["op_p"]), atol=1e-5)
        np.testing.assert_allclose(skp[a], fw["skip_p"], atol=1e-5)
    for l in range(L):
        obs = np.bincount(arcs[:, l * (l + 1) // 2], minlength=n_ops)
        exp = opp[:, l, :].astype(np.float64).sum(axis=0)
        exp *= obs.sum() / exp.sum()
        assert ss.chisquare(obs, exp).pvalue > 1e-4, (l, obs, exp)
    pos = [l * (l + 1) // 2 + 1 + j for l in range(1, L) for j in range(l)]
    x = arcs[:, pos].astype(np.float64)
    p = skp.astype(np.float64)
    z = (x.sum() - p.sum()) / np.sqrt((p * (1 - p)).sum())
    assert abs(z) < 4.5, z
    assert len(np.unique(arcs, axis=0)) > 100
    ctl.close()


def test_determinism():
    outs = []
    for _ in range(2):
        ctl = _controller(12, 64, 78, O.settings(learning_rate=0.01), seed=42)
        a1 = ctl.sample(16)
        s1 = ctl.train(0.5, 20)
        a2 = ctl.sample(300)
        s2 = ctl.train(0.9, 7)
        st = ctl.state()
        outs.append((a1, s1, a2, s2, st))
        ctl.close()
    (a, b) = outs
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    for key in ("params", "m", "v"):
        for n in O.PARAM_NAMES:
            assert np.array_equal(a[4][key][n], b[4][key][n])
    assert a[4]["baseline"] == b[4]["baseline"] and a[4]["step"] == b[4]["step"] == 27 and a[4]["draws"] == b[4]["draws"] == 29


def test_bad_imposed_arc_is_refused():
    from kubeflow_b200._lib import KboInvalidArgument
    ctl = _controller(3, 8, 4, O.settings())
    bad = np.zeros((1, 6), np.int32)
    bad[0, 3] = 4
    with pytest.raises(KboInvalidArgument):
        ctl.train(1.0, 1, arcs=bad)
    assert ctl.state()["step"] == 0
    ctl.close()


def test_controllers_of_different_shapes_coexist():
    """The kernels' shared-memory limit is process-wide: creating a small controller after a large one must leave the large
    one able to train and sample."""
    st = O.settings()
    big = _controller(64, 128, 4096, st, seed=5)
    mid = _controller(8, 64, 78, st, seed=6)
    small = _controller(1, 1, 1, st, seed=7)
    for ctl in (big, mid, small, big):
        stats = ctl.train(0.5, 2)
        arcs = ctl.sample(5)
        assert np.isfinite(stats).all() and arcs.shape == (5, ctl.A)
    assert big.state()["step"] == 4 and small.state()["step"] == 2
    for ctl in (big, mid, small):
        ctl.close()


def test_draw_at_u_one_takes_the_last_op_with_weight():
    """u = 1 leaves u·total at the total, so no prefix sum exceeds it: the draw falls back to the last op whose weight did not
    underflow (here op 3: op 4's logit is about -3000 with no tanh or temperature to bound it)."""
    st = O.settings(temperature=None, tanh_const=None)
    ctl = _controller(1, 4, 5, st)
    P = {n: np.zeros_like(a) for n, a in ctl.state()["params"].items()}
    P["g_emb"][:] = 1.0
    P["w_lstm"][:4, :] = 10.0                               # x = g_emb drives every gate open: h = tanh(1) > 0
    P["w_soft"][:, 4] = -1000.0
    ctl.set_params(P)
    arcs, opp, _ = ctl.sample(3, uniforms=np.array([[1.0], [0.5], [0.0]], np.float32), return_probs=True)
    assert opp[0, 0, 4] == 0.0 and arcs[:, 0].tolist() == [3, 2, 0]
    p64 = O.forward({n: a.astype(np.float64) for n, a in ctl.state()["params"].items()}, 1, st, arc=[0])["op_p"][0]
    assert [O.draw(p64, u) for u in (1.0, 0.5, 0.0)] == [3, 2, 0]
    ctl.close()


def test_reinforce_raises_the_probability_of_rewarded_arcs():
    """End to end on the GPU: steps whose arcs all take op 0 at every layer, with a reward above the baseline (the
    advantage is positive), raise op 0's probability at every layer; with the reward below the baseline they lower it.  The
    skip penalty and the entropy bonus are off, so only the REINFORCE term moves the controller."""
    L, H, n_ops = 4, 16, 6
    arcs = np.zeros((30, L * (L + 1) // 2), np.int32)
    for sign in (1.0, -1.0):
        ctl = _controller(L, H, n_ops, O.settings(learning_rate=0.01, skip_weight=None, entropy_weight=None), seed=9)
        before = ctl.sample(1, uniforms=np.zeros((1, L * (L + 1) // 2), np.float32), return_probs=True)[1][0, :, 0]
        ctl.set_params(ctl.state()["params"], baseline=-sign * 1.0)
        ctl.train(0.0, 30, arcs=arcs)
        after = ctl.sample(1, uniforms=np.zeros((1, L * (L + 1) // 2), np.float32), return_probs=True)[1][0, :, 0]
        print(f"advantage sign {sign:+.0f}: P(op 0) per layer {before.round(4).tolist()} -> {after.round(4).tolist()}")
        assert (np.sign(after - before) == sign).all(), (sign, before, after)
        ctl.close()


# ---------------------------------------------------------------------------------------------------------------- service
from tests.test_enas_service import make_experiment  # noqa: E402


@pytest.fixture()
def stub():
    from kubeflow_b200.suggestion.enas_service import EnasService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    svc = EnasService()
    server, port = serve(svc, port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


SERVICE_SETTINGS = {"random_state": 17, "controller_hidden_size": 32, "controller_learning_rate": 0.01, "controller_train_steps": 10,
                    "controller_baseline_decay": 0.9}


def _rounds(s, name, n_rounds, settings=SERVICE_SETTINGS, layers=5):
    from kubeflow_b200.suggestion import api_pb as api
    exp = make_experiment(settings, name=name, num_layers=layers)
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=4)
    replies, rewards = [], []
    for r in range(n_rounds):
        rep = s.GetSuggestions(req)
        arcs = [json.loads(pa.assignments[0].value.replace("'", '"')) for pa in rep.parameter_assignments]
        replies.append(arcs)
        for i, arc in enumerate(arcs):
            t = req.trials.add()
            t.name = f"{name}-{r}-{i}"
            t.status.condition = api.SUCCEEDED
            m = t.status.observation.metrics.add()
            m.name, m.value = "accuracy", repr(float(np.mean([layer[0] == 0 for layer in arc])))
        rewards.append(np.mean([float(t.status.observation.metrics[0].value) for t in req.trials]))
    return replies, rewards


def test_service_rounds_match_the_oracle(stub):
    from kubeflow_b200.suggestion.enas_service import validate_enas_settings
    s, svc = stub
    L, n_ops = 5, 6                                         # make_experiment's space expands to 6 operations
    replies, rewards = _rounds(s, "enas-parity", 20)
    st_set = validate_enas_settings({k: str(v) for k, v in SERVICE_SETTINGS.items()})
    st = O.settings(**{k: st_set["controller_" + k] for k in O.settings()})
    eng = svc._exps["enas-parity"].engine
    from kubeflow_b200.enas import EnasController
    fresh = EnasController(L, 32, n_ops, settings=st, seed=17)
    ref = O.new_state(fresh.state()["params"])
    fresh.close()
    seed, draw, T = 17, 0, SERVICE_SETTINGS["controller_train_steps"]
    for r in range(20):
        if r > 0:                                           # R: the mean over every SUCCEEDED trial sent so far
            for _ in range(T):
                u = [O.philox_uniform(seed, draw, 0, d) for d in range(L * (L + 1) // 2)]
                O.train_step(ref, L, st, rewards[r - 1], uniforms=u)
                draw += 1
        for a, arc in enumerate(replies[r]):
            u = [O.philox_uniform(seed, draw, a, d) for d in range(L * (L + 1) // 2)]
            want = O.organise_arc(O.forward(ref["params"], L, st, uniforms=u)["arc"], L)
            assert arc == want, (r, a, arc, want)
        draw += 1
    got = eng.state()
    for n in O.PARAM_NAMES:
        assert np.abs(got["params"][n] - ref["params"][n]).max() <= 1e-5, n
    assert abs(got["baseline"] - ref["baseline"]) <= 1e-5 and got["step"] == 19 * T


def test_two_fresh_services_reply_identically():
    from kubeflow_b200.suggestion.enas_service import EnasService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    out = []
    for _ in range(2):
        server, port = serve(EnasService(), port=0, host="127.0.0.1")
        ch = grpc.insecure_channel(f"127.0.0.1:{port}")
        out.append(_rounds(SuggestionStub(ch), "enas-twin", 4)[0])
        ch.close()
        server.stop(0)
    assert out[0] == out[1]


def test_changed_nas_config_gives_a_fresh_controller(stub):
    from kubeflow_b200.suggestion import api_pb as api
    s, svc = stub
    _rounds(s, "enas-swap", 3)
    old = svc._exps["enas-swap"]
    assert old.engine.state()["step"] == 2 * SERVICE_SETTINGS["controller_train_steps"]
    rep = s.GetSuggestions(api.GetSuggestionsRequest(experiment=make_experiment(SERVICE_SETTINGS, name="enas-swap", num_layers=3),
                                                     current_request_number=2))
    new = svc._exps["enas-swap"]
    assert new is not old and new.engine.L == 3 and new.engine.state()["step"] == 0 and len(rep.parameter_assignments) == 2
    assert all(len(json.loads(pa.assignments[0].value.replace("'", '"'))) == 3 for pa in rep.parameter_assignments)
