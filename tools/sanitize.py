"""Small end-to-end invocations of every kernel for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from kubeflow_b200.gp import GPEngine
from kubeflow_b200.cmaes import CmaEs


def synthetic(N, M, D):
    """The workload of record (SURVEY.md §8(d)), restated here so that tools/ never touches oracle/."""
    X = np.random.default_rng(1234).random((N, D))
    y = np.sin(3.0 * X.sum(axis=1) / np.sqrt(D)) + 0.1 * np.random.default_rng(1235).standard_normal(N)
    Xc = np.random.default_rng(4321).random((M, D))
    return X, y, Xc


def theta_of_record(D):
    return dict(length_scale=0.3 * np.sqrt(D), amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96)


for N, M, D, mode in ((70, 300, 3, "f64"), (135, 515, 5, "tc"), (300, 700, 33, "tc"), (700, 1900, 40, "tc"),   # 700: 2 tile pairs -> pruning pass
                      (1100, 2500, 12, "tc")):   # 1100: lazy inverse (leading 512 rows of W), alpha and survivors by the cooperative panel solves, 5 panels of the look-ahead factorisation
    X, y, Xc = synthetic(N, M, D)
    th = theta_of_record(D)
    e = GPEngine(0, kernel="matern52", acq="ei", var_mode=mode, **th)
    e.tell(X, y)
    b = e.ask(Xc.astype(np.float32))
    b2, t = e.suggest_host(X, y, Xc)
    e.tell(X[:N - 3], y[:N - 3])                 # bordered-Cholesky appends, a rebase, the FP64 refinement of the tc pick, LML gradient
    for i in range(N - 3, N):
        e.append(X[i], y[i])
    b3 = e.ask(Xc)
    e.rebase(N - 5, y[:N - 5] * 0.5)
    b4 = e.ask(Xc)
    g = e.lml_grad()[1]
    lm = e.lml_batch(X, y, [dict(noise=1e-3), dict(noise=1e-2, length_scale=th["length_scale"] * 2)])
    lg = e.lml_grad_batch(X, y, [dict(noise=1e-3), dict(noise=0.0, amplitude=2.0)])      # lanes with W, K⁻¹ and the gradient
    b5, _, _, _ = e.ask(Xc, return_arrays=True)      # three-product / FP64 array path
    print(N, M, D, mode, b.index, b2.index, b3.index, b4.index, b5.index, e.last_contenders(), e.last_prefix_survivors(), float(g[0]), lm.tolist(), lg[0].tolist())
    e.close()
    if mode == "tc":                                  # the ranking pass without pruning, and the round-1 ranking pass
        for kw in (dict(rank_prefix=0), dict(rank_tc=False)):
            e = GPEngine(0, kernel="matern52", acq="ei", var_mode=mode, **th, **kw)
            e.tell(X, y)
            print("   ", kw, e.ask(Xc.astype(np.float32)).index)
            e.close()
es = CmaEs(np.zeros(9), 1.0, popsize=20, seed=1)
print(es.run_synthetic("sphere", 3))
es.set_lr_adapt(True)                                # LRA tells: prep, three products, the blend, the finish
print(es.run_synthetic("rastrigin", 3), es.lr_state()["eta_mean"])
es.restart(40, np.full(9, 0.5), 0.3)                 # an LRA restart with a larger λ, then a tell of the new run
print(es.run_synthetic("sphere", 2), es.lr_state()["eta_mean"])
es.close()
from kubeflow_b200.cmaes import SepCmaEs              # separable CMA-ES: two CTAs of the update at D = 300, a restart to a larger λ
for D, lam in ((9, 20), (300, 16)):
    es = SepCmaEs(np.zeros(D), 1.0, popsize=lam, seed=1)
    for _ in range(3):
        X = es.ask()
        es.tell((X * X).sum(1))
    es.restart(2 * lam, np.full(D, 0.5), 0.3)
    X = es.ask()
    es.tell((X * X).sum(1))
    print(D, lam, es.stop_flags()[0], es.state()["sigma"])
    es.close()
from kubeflow_b200.tpe import Tpe                     # TPE: model build (radix + segmented sorts), draws, FP32 score + FP64 decision, levels
_r = np.random.default_rng(3)
tp = Tpe([("uniform", -1.0, 3.0), ("quniform", 3.0, 48.0, 5.0), ("choice", 5), ("quniform", 0.0, 1e6, 1.0)], seed=9)
tp.tell(np.c_[_r.uniform(-1, 3, 300), 5.0 * _r.integers(1, 10, 300), _r.integers(0, 5, 300), _r.integers(0, 10 ** 6, 300)], _r.random(300))
print(tp.ask(2, 3000).tolist(), tp.last_survivors().tolist(), tp.state()[0]["below"]["w"].shape)
tp.close()
from kubeflow_b200.mvtpe import MvTpe                 # multivariate TPE: model build, tables, draws, prep, FP32 score + FP64 decision
mv = MvTpe([("float", -1.0, 3.0), ("int", 3, 48, 5), ("cat", 5), ("int", 0, 10 ** 6, 1), ("float", 0.0, 1.0)], seed=9)
mv.tell(np.c_[_r.uniform(-1, 3, 300), 3.0 + 5.0 * _r.integers(0, 10, 300), _r.integers(0, 5, 300), _r.integers(0, 10 ** 6, 300), _r.random(300)],
        _r.random(300))
print(mv.ask(2, 300).tolist(), mv.last_survivors().tolist(), mv.state()["below"]["w"].shape)
mv.close()
_wide = [("float", 0.0, 1.0)] * 40 + [("int", 0, 19, 1), ("cat", 3)] * 10     # two float slabs, two discrete slabs in the score kernel
mv = MvTpe(_wide, seed=3)
mv.tell(np.c_[_r.random((300, 40)), np.column_stack([_r.integers(0, 20 if i % 2 == 0 else 3, 300) for i in range(20)])], _r.random(300))
print(mv.ask(2, 300).shape, mv.last_survivors().tolist())
mv.close()
from kubeflow_b200.forest import ForestEngine       # RF / ET: bootstrap, presort, per-tree fit, packing, staged sweep, export draws
for _kind in ("RF", "ET"):
    fe = ForestEngine(kind=_kind, n_trees=8, seed=4)
    fe.tell(_r.random((300, 5)), _r.random(300))
    print(fe.ask_multi(_r.random((5000, 5)), ["ei", "lcb", "pi"])[0], fe.predict(_r.random((3, 5)))[0].tolist(),
          len(fe.export(0, with_draws=_kind == "ET")["left"]))
    fe.close()
from kubeflow_b200.gbrt import GbrtEngine           # GBRT: init, presort, the three-chain fit, staged sweep and predict, export
ge = GbrtEngine()
ge.tell(_r.random((300, 5)), _r.random(300))
print(ge.ask_multi(_r.random((5000, 5)), ["ei", "lcb", "pi"])[0], ge.predict(_r.random((3, 5)), return_std=True)[1].tolist(),
      len(ge.export(2, 29)["left"]))
ge.close()
from kubeflow_b200.enas import EnasController        # ENAS: init, the one-CTA train chain (drawn and imposed arcs), batched draws
en = EnasController(5, 12, 9, seed=2)
print(en.sample(6).tolist(), en.train(0.5, 3)[:, 0].tolist())
print(en.train(0.7, 2, arcs=en.sample(2)).shape, en.sample(5, uniforms=_r.random((5, 15)), return_probs=True)[0].tolist())
en.close()


def refused(call):                                   # a call that fails after it has allocated: nothing may leak
    try:
        call()
    except ValueError as ex:
        return str(ex).splitlines()[0][:60]
    raise AssertionError("the call was expected to be refused")


tp = Tpe([("uniform", -1.0, 3.0), ("choice", 5)], seed=1)    # history grown twice (64 -> 128 -> 256 rows), the told rows kept
for n in (40, 40, 100):
    tp.tell(np.c_[_r.uniform(-1, 3, n), _r.integers(0, 5, n)], _r.random(n))
bad = torch.zeros(1, 2, 64, dtype=torch.float64, device="cuda:0")
bad[0, 1, 7] = 9.0                                    # category 9 of 5
print(tp.ask(1, 64).tolist(), refused(lambda: tp.ask(1, 64, candidates=bad)))
tp.close()
mv = MvTpe([("float", 0.0, 1.0), ("cat", 3)], seed=1)
mv.tell(np.c_[_r.random(20), _r.integers(0, 3, 20)], _r.random(20))
print(refused(lambda: mv.tell([[0.5, 1.0]], [float("nan")])), mv.ask(1, 64).tolist())
mv.close()
fe = ForestEngine(kind="RF", n_trees=4, seed=1)
Xn = _r.random((50, 3))
Xn[7, 1] = np.nan
print(refused(lambda: fe.tell(Xn, _r.random(50))))
fe.close()
