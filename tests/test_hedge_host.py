"""CPU: gp_hedge (Katib's default acquisition) in the Optimizer's host logic, against a replay built on oracle/hedge_oracle.py —
skopt's bookkeeping restated.  The engine is the oracle-backed stand-in of test_spmd_gloo with the two calls gp_hedge needs
(ask_multi, predict_mean); the GPU engine's versions of those are checked in test_gpu_hedge.py.  Covered: the random phase,
the first model-based ask, a re-ask with no new trials (gains unchanged), new trials (gains advance once), ask(n_points=3)
(the lies advance a scratch copy only), a MAXIMIZE objective through the service, and a sharded optimizer over gloo."""
import os
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Integer, Real
from oracle import gp_oracle as O
from oracle.hedge_oracle import HedgeOracle
from tests.test_spmd_gloo import OracleEngine


class HedgeOracleEngine(OracleEngine):
    """OracleEngine plus ask_multi / predict_mean; records every ask_multi call (offset, candidates, history)."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def _fit(self):
        return O.gp_fit(self.X, self.y, kind=self.kernel, length_scale=self.length_scale, amplitude=self.amplitude, noise=self.noise)

    def ask_multi(self, cand, acqs, global_offset=0):
        from kubeflow_b200.gp import Best
        cand = np.asarray(cand, dtype=np.float64)
        mu, std = O.gp_predict(self._fit(), cand)
        out = []
        for a in acqs:
            v = O.acquisition(mu, std, float(np.min(self.y)), a, self.xi, self.kappa)
            i = O.first_argmax(v)
            out.append(Best(float(v[i]), global_offset + i, float(mu[i]), float(std[i])))
        self.calls.append((global_offset, cand, self.X.copy(), self.y.copy()))
        return out

    def predict_mean(self, X):
        return O.gp_predict(self._fit(), np.atleast_2d(np.asarray(X, dtype=np.float64)))[0]


class Replay:
    """The Optimizer's sequence of draws and tells, replayed on HedgeOracle with the repository's rules: the gains advance on
    the first model-based ask after the told history changed; lies work on a copy that starts from the told step's picks."""

    def __init__(self, space, seed, n_initial_points, n_points):
        self.space, self.n_init, self.n_points = space, n_initial_points, n_points
        self.rng = np.random.default_rng(seed)
        self.real = HedgeOracle(length_scale=0.3 * np.sqrt(space.transformed_n_dims))
        self.hist = None

    def ask(self, Xt, y, k=1):
        Xt, y, out, copy = np.asarray(Xt, dtype=np.float64).reshape(len(y), self.space.transformed_n_dims), list(y), [], None
        for i in range(k):
            if len(y) < max(self.n_init, 1):
                row, gp = self.space.rvs_transformed(1, self.rng, np.float64)[0], False
            else:
                cand = self.space.rvs_transformed(self.n_points, self.rng, np.float32)
                ya = np.asarray(y, dtype=np.float64)
                if i == 0:
                    h = self.hist
                    changed = h is None or h[0].shape != Xt.shape or not (np.array_equal(h[0], Xt) and np.array_equal(h[1], ya))
                    row = self.real.tell(Xt, ya, cand, self.rng, update=changed)[0]
                    self.hist = (Xt.copy(), ya.copy())
                else:
                    row = copy.tell(Xt, ya, cand, self.rng)[0]
                gp = True
            if i == 0:
                copy = self.real.copy()
                if gp:
                    copy.next_xs = self.real.next_xs
            x = self.space.inverse_transform(np.asarray(row, dtype=np.float64)[None, :])[0]
            out.append(x)
            if y:
                Xt = np.concatenate([Xt, self.space.transform([x])])
                y.append(min(y))
        return out


def _dims():
    return [Real(0.0, 1.0, name="a"), Real(-2.0, 2.0, name="b"), Integer(1, 9, name="c")]


def _f(p):
    return float(np.sin(3 * p[0]) + 0.3 * p[1] ** 2 + 0.05 * p[2])


def _check(opt, rep, got, want):
    assert got == want
    np.testing.assert_allclose(opt.gains, rep.real.gains, rtol=0, atol=1e-12)
    if rep.real.next_xs is None:
        assert opt.next_xs is None
    else:
        np.testing.assert_array_equal(opt.next_xs, rep.real.next_xs)


def test_hedge_picks_and_gains_follow_skopt():
    eng = HedgeOracleEngine()
    opt = Optimizer(_dims(), n_initial_points=3, acq_func="gp_hedge", random_state=7, n_points=400, candidate_backend="numpy", engine=eng)
    rep = Replay(opt.space, 7, 3, 400)
    told_X, told_y = [], []

    def tell(pts):
        ys = [_f(p) for p in pts]
        opt.tell(pts, ys)
        told_X.extend(pts)
        told_y.extend(ys)

    def ask(k=None):
        got = opt.ask() if k is None else opt.ask(n_points=k)
        want = rep.ask(opt.space.transform(told_X) if told_X else np.empty((0, 0)), told_y, 1 if k is None else k)
        _check(opt, rep, got if k is not None else [got], want)
        return got if k is not None else [got]

    asks = 0
    tell(ask()); asks += 1                                  # random phase: no gains, no picks
    assert opt.next_xs is None and not opt.gains.any()
    tell(ask(2)); asks += 2                                 # still random (lies count toward the history)
    ask(); asks += 1                                        # first model-based ask: picks, no update yet
    assert opt.next_xs is not None and not opt.gains.any()
    g0 = opt.gains.copy()
    ask(); asks += 1                                        # re-ask, no new trials: the gains do not move
    np.testing.assert_array_equal(opt.gains, g0)
    pts = ask(3); asks += 3                                 # batch: the real step sees no new trials, the lies use a copy
    np.testing.assert_array_equal(opt.gains, g0)
    assert eng.log.count("append") >= 2
    tell(pts)
    ask(); asks += 1                                        # new trials: the gains advance once
    assert opt.gains.any()
    g1 = opt.gains.copy()
    ask(); asks += 1
    np.testing.assert_array_equal(opt.gains, g1)
    tell(ask(3)[:2]); asks += 3                             # the real step sees no new trials: g1 stays
    np.testing.assert_array_equal(opt.gains, g1)
    ask(); asks += 1
    assert not np.array_equal(opt.gains, g1)
    ask(); asks += 1
    assert asks >= 15


def test_a_failed_sweep_does_not_advance_the_gains():
    """An ask whose sweep raises leaves the gains and picks as they were and makes the next ask refit; the retry then advances
    the gains exactly once, as an ask that never failed does."""
    def run(fail):
        eng = HedgeOracleEngine()
        opt = Optimizer(_dims(), n_initial_points=3, acq_func="gp_hedge", random_state=9, n_points=300, candidate_backend="numpy", engine=eng)
        r = np.random.default_rng(2)
        X = [[float(r.random()), float(r.uniform(-2, 2)), int(r.integers(1, 10))] for _ in range(5)]
        opt.tell(X, [_f(p) for p in X])
        opt.ask()
        opt.tell([X[0]], [0.3])
        if fail:
            real = eng.ask_multi
            eng.ask_multi = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("sweep failed"))
            g, nx = opt.gains.copy(), opt.next_xs.copy()
            try:
                opt.ask()
                raise AssertionError("the sweep should have raised")
            except RuntimeError:
                pass
            np.testing.assert_array_equal(opt.gains, g)
            np.testing.assert_array_equal(opt.next_xs, nx)
            assert opt._fit_state is None
            eng.ask_multi = real
        opt.ask()
        return opt.gains.copy()

    ok, failed = run(False), run(True)
    assert ok.any()
    np.testing.assert_array_equal(failed, ok)


def test_hedge_through_the_service_with_a_maximize_objective():
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.service import SkoptService
    from tests.test_grpc_service import add_trial, make_experiment
    eng = HedgeOracleEngine()
    svc = SkoptService({"engine": eng, "candidate_backend": "numpy"})
    exp = make_experiment("bayesianoptimization", {"n_initial_points": 4, "random_state": 3, "n_points": 300}, objective=api.MAXIMIZE, name="hedge-max")
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=2)
    metric = lambda v: -((v["x0"] - 0.05) ** 2 * 100 + v["x1"] ** 2 + ((v["x2"] - 15) / 5) ** 2 + ((v["x3"] - 2) / 2) ** 2)
    rep, n, told = None, 0, []
    for r in range(5):
        rp = svc.get_suggestions(req)
        opt = svc._services["hedge-max"].skopt_optimizer
        assert opt.hedge                                      # the default acq_func is gp_hedge
        if rep is None:
            rep = Replay(opt.space, 3, 4, 300)
        pts = [[float(a.value) for a in pa.assignments] for pa in rp.parameter_assignments]
        Xt = opt.space.transform([p for p, _ in told]) if told else np.empty((0, 0))
        want = rep.ask(Xt, [-m for _, m in told], 2)          # the service tells the loss: −metric for MAXIMIZE
        for p, w in zip(pts, want):
            np.testing.assert_array_equal(p, w)
        np.testing.assert_allclose(opt.gains, rep.real.gains, rtol=0, atol=1e-12)
        for p in pts:
            v = dict(zip(["x0", "x1", "x2", "x3"], p))
            n += 1
            add_trial(req, f"t{n}", v, metric(v))
            told.append((p, metric(v)))
    assert opt.yi == [-m for _, m in told[:len(opt.yi)]]
    assert opt.gains.any()


# ---- sharded, world size 2 over gloo --------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    eng = HedgeOracleEngine()
    opt = Optimizer(_dims(), n_initial_points=3, acq_func="gp_hedge", random_state=5, n_points=401, candidate_backend="numpy", engine=eng,
                    shard=True)
    r = np.random.default_rng(1)
    X = [[float(r.random()), float(r.uniform(-2, 2)), int(r.integers(1, 10))] for _ in range(6)]
    opt.tell(X, [_f(p) for p in X])
    out = [opt.ask()]
    opt.tell(out[-1:], [_f(out[-1])])
    out += opt.ask(n_points=2)
    opt.tell(out[-2:], [_f(p) for p in out[-2:]])
    out.append(opt.ask())
    bests, _, j = opt.last_hedge
    goff, cand, Xh, yh = eng.calls[-1]
    q.put(dict(rank=rank, out=out, gains=opt.gains.tolist(), idx=[b.index for b in bests], vals=[b.value for b in bests], j=j,
               next_xs=opt.next_xs.tolist(), goff=goff, cand=cand, Xh=Xh, yh=yh))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_hedge_two_ranks_over_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted([q.get(timeout=300) for _ in ps], key=lambda d: d["rank"])
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    r0, r1 = res
    assert r0["out"] == r1["out"] and r0["gains"] == r1["gains"] and r0["j"] == r1["j"]
    assert any(g != 0.0 for g in r0["gains"])
    assert r0["goff"] == 0 and r1["goff"] == 201 and len(r0["cand"]) == 201 and len(r1["cand"]) == 200
    np.testing.assert_array_equal(r0["Xh"], r1["Xh"])
    cand = np.concatenate([r0["cand"], r1["cand"]])
    fit = O.gp_fit(r0["Xh"], r0["yh"], length_scale=0.3 * np.sqrt(3), noise=1e-3)
    mu, std = O.gp_predict(fit, cand)
    for k, a in enumerate(("ei", "lcb", "pi")):
        i = O.first_argmax(O.acquisition(mu, std, float(np.min(r0["yh"])), a))
        assert r0["idx"][k] == r1["idx"][k] == i
        np.testing.assert_array_equal(r0["next_xs"][k], cand[i])
        np.testing.assert_array_equal(r1["next_xs"][k], cand[i])
