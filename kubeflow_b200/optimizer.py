"""``Optimizer`` — the host-side mirror of ``skopt.Optimizer`` as Katib's skopt service drives it
(upstream kubeflow/katib pkg/suggestion/v1beta1/skopt/base_service.py: ``tell(X, y)`` then ``ask()`` per
requested assignment).  Differences, stated once:

* θ is FIXED per request by default (length scales, amplitude, noise are settings), where skopt refits them by L-BFGS on the
  log-marginal likelihood ($SK/_gpr.py:299-339).  ``theta_fit="skopt"`` fits θ as skopt does (``kubeflow_b200.thetafit``):
  amplitude, ARD length scales and noise over skopt's bounds, by SciPy's L-BFGS-B from 1 + ``theta_restarts`` (default 2)
  starts drawn as sklearn draws them, run in lockstep with one ``GPEngine.lml_grad_batch`` call per round; the engine is then
  fitted at the winner.  θ is refitted once per change of the told history; constant-liar lies reuse it and take the append
  path, where skopt refits θ on each lie's copy.  ``kernel="rbf"`` is allowed there.  An all-categorical space keeps
  Matérn on its one-hot columns by default, where skopt switches to a HammingKernel; ``kernel="hamming"`` gives skopt's
  model there (``kubeflow_b200.hamming``): θ holds the per-dimension weights l_j (``length_scale`` is the isotropic l, 1.0 by
  default; ``theta_fit="skopt"`` fits one l_j per dimension over (1e-5, 1e5)), mapped to RBF length scales of the one-hot
  columns in one place, so the fit, append, rebase, sweep and LML gradient are the engine's own.  It is refused, before any
  device is touched, unless every dimension is Categorical, and beside ``theta_grid``, ``theta_search`` or
  ``theta_fit="lbfgs"``, which search one-hot length scales.  Older GPU-side substitutes, both maximising
  the device-computed LML (one FP64 fit per candidate θ):
  ``theta_grid`` = G > 1 tries G multiples of the length scale (geometric, 0.25×…4×); ``theta_search`` = K > 0 additionally
  draws K random (length-scale multiple, noise) pairs log-uniformly from [0.2, 5] × [1e-6, 1e-1] (seeded) — the gradient-free
  analogue of skopt's restarts; ``theta_fit="lbfgs"`` then polishes (log ℓ — per dimension with ``ard=True`` —, log noise)
  with SciPy's L-BFGS-B exactly as sklearn does ($SK/_gpr.py:658-667), every objective/gradient evaluation being one
  device fit + ``kbo_lml_grad`` (SURVEY.md §8(f)1).
* ``acq_optimizer`` is "sampling" over ``n_points`` candidates (skopt default 10 000; here 65 536 by default and
  millions are cheap) — ``lbfgs`` polishing is accepted by ValidateAlgorithmSettings and mapped to sampling; ``EIps`` /
  ``PIps`` (they need a second model of the trial durations) are mapped to EI / PI.
* ``ask(n_points=k)`` uses skopt's constant-liar "cl_min" strategy: k sequential asks with the lie y = min(y).
* ``base_estimator`` "RF" / "ET" use skopt's forests (``kubeflow_b200.forest.ForestEngine``: fit and sweep on the GPU, raw y, no
  θ), refit whenever the history changes — every lie included — and swept over the same candidates, shards, gp_hedge and
  constant liar as the GP.  Their seed is fixed when the engine is made.
* GBRT is served when ``base_estimator`` is a ``kubeflow_b200.gbrt.GbrtEngine`` **instance**, the way skopt's ``gbrt_minimize``
  passes a ``GradientBoostingQuantileRegressor`` instance; it takes the forests' path (raw y, a refit for every lie, gp_hedge,
  shards) and stays the caller's: ``close()`` does not close it.  The string ``"GBRT"`` is refused.

``acq_func="gp_hedge"`` (Katib's and skopt's default) is skopt's portfolio: every model-based ask sweeps ONE candidate set
for EI, LCB and PI together (``GPEngine.ask_multi``: one posterior, three first-index argmaxes), keeps the three picks, and
draws which one to suggest from softmax(η·gains), η = 1.  When the history has changed, the next model-based ask first
subtracts the new model's posterior mean (raw y scale, ``GPEngine.predict_mean``) at the previous three picks from the
gains — skopt's ``gains_ -= est.predict(vstack(next_xs_))``, a pick that turned out well predicted low gaining most.
Here ``tell`` is lazy and the work happens in ``ask``, so:

* the gains advance once per change of the told history: on the first model-based ask after new trials, with the picks
  of the last sweep on the told history; an ask with no new trials leaves them alone;
* during the ``n_initial_points`` random phase there are no gains updates and no picks;
* in ``ask(n_points=k)`` the first point is the told-history step; points 2..k come from the lie-extended histories with a
  scratch copy of the gains that advances once per lie, as the copy skopt's ``ask`` works on does — the real gains never
  see a lie;
* the draw uses ``self.rng`` (a NumPy Generator), so every rank of a sharded optimizer draws the same.

Against skopt's gp_hedge, besides the fixed θ and the candidate count above: the draw comes from a NumPy Generator, not
a RandomState, and the first point of a batch is the told-history step's draw, where skopt redraws it on its copy.
"""
from __future__ import annotations

import numpy as np

from .space import Space


HEDGE_ACQS = ("ei", "lcb", "pi")   # skopt's cand_acq_funcs_ = ["EI", "LCB", "PI"]
FOREST_ESTIMATORS = ("RF", "ET")   # skopt's cook_estimator forests, kubeflow_b200.forest.ForestEngine


class Optimizer:
    def __init__(self, dimensions, base_estimator="GP", n_initial_points=10, acq_func="EI", acq_optimizer="sampling",
                 random_state=None, *, n_points=65536, kernel="matern52", length_scale=None, amplitude=1.0, noise=1e-3, xi=0.01,
                 kappa=1.96, var_mode="auto", theta_grid=1, theta_search=0, theta_fit=None, theta_fit_maxiter=None, theta_restarts=None, ard=False,
                 device=0, engine=None, candidate_backend="torch", incremental=True, shard=False):
        self._gbrt = None             # a GbrtEngine passed as base_estimator (owned by the caller)
        if isinstance(base_estimator, str):
            self.base_estimator = base_estimator.upper()
            if self.base_estimator not in ("GP",) + FOREST_ESTIMATORS:
                raise ValueError("base_estimator must be GP, RF or ET, or a kubeflow_b200.gbrt.GbrtEngine instance for GBRT")
        else:
            from .gbrt import GbrtEngine
            if not isinstance(base_estimator, GbrtEngine):
                raise ValueError(f"base_estimator must be GP, RF, ET or a GbrtEngine instance, got {type(base_estimator).__name__}")
            self._gbrt, self.base_estimator = base_estimator, "GBRT"
        self.forest = self.base_estimator in FOREST_ESTIMATORS + ("GBRT",)   # the tree path: raw y, refit on every change
        if self.forest and acq_optimizer == "lbfgs":
            name = {"RF": "RandomForestRegressor", "ET": "ExtraTreesRegressor", "GBRT": "GradientBoostingQuantileRegressor"}[self.base_estimator]
            raise ValueError(f"The regressor {name} should run with acq_optimizer='sampling'.")
        self.space = dimensions if isinstance(dimensions, Space) else Space(dimensions)
        self.n_initial_points = int(n_initial_points)
        acq = str(acq_func)
        self.acq = {"EI": "ei", "LCB": "lcb", "PI": "pi", "gp_hedge": "ei", "EIps": "ei", "PIps": "pi"}.get(acq)
        if self.acq is None:
            raise ValueError(f"unknown acq_func {acq_func!r}")
        # gp_hedge portfolio state (host-only: constructing a hedge optimizer touches no device)
        self.hedge = acq == "gp_hedge"
        self.eta = 1.0
        self.gains = np.zeros(len(HEDGE_ACQS)) if self.hedge else None
        self.next_xs = None           # transformed rows of the last told-history sweep's EI / LCB / PI picks
        self._hedge_hist = None       # (Xt, y) those picks were made on
        self._lie_gains = self._lie_next_xs = None   # scratch state of the lies of one ask(n_points=k)
        self._last_gp = False         # the last _ask_one was model-based
        self.last_hedge = None        # (Bests of EI / LCB / PI, probabilities, index drawn) of the last hedge ask
        if acq_optimizer not in ("auto", "sampling", "lbfgs"):
            raise ValueError(f"unknown acq_optimizer {acq_optimizer!r}")
        self.rng = np.random.default_rng(random_state)
        self.n_points = int(n_points)
        self.kernel, self.amplitude, self.noise, self.xi, self.kappa = kernel, amplitude, noise, xi, kappa
        self.length_scale = length_scale
        self.var_mode, self.theta_grid, self.theta_search, self.device = var_mode, int(theta_grid), int(theta_search), device
        if theta_fit not in (None, "lbfgs", "skopt"):
            raise ValueError("theta_fit must be None, 'lbfgs' or 'skopt'")
        if theta_restarts is not None and theta_fit != "skopt":
            raise ValueError("theta_restarts applies to theta_fit='skopt' only")
        if theta_fit == "skopt":      # the start and the fit are skopt's: nothing may set or search θ beside it
            for name, given in (("theta_grid", int(theta_grid) > 1), ("theta_search", int(theta_search) > 0), ("ard", bool(ard)),
                                ("length_scale", length_scale is not None), ("amplitude", amplitude != 1.0), ("noise", noise != 1e-3)):
                if given:
                    raise ValueError(f"{name} cannot be combined with theta_fit='skopt': skopt's start and bounds are used")
            if theta_restarts is not None and int(theta_restarts) < 0:
                raise ValueError(f"theta_restarts must be >= 0, got {theta_restarts}")
        self._hmap = None             # kernel="hamming": the map from Hamming weights to the one-hot columns' RBF θ
        if kernel == "hamming":
            from .hamming import HammingMap
            self._hmap = HammingMap(self.space)
            for name, given in (("theta_grid", int(theta_grid) > 1), ("theta_search", int(theta_search) > 0),
                                ("theta_fit='lbfgs'", theta_fit == "lbfgs")):
                if given:
                    raise ValueError(f"{name} cannot be combined with kernel='hamming': it searches one-hot length scales")
        self.theta_fit, self.ard = theta_fit, bool(ard)
        self.theta_fit_maxiter = None if theta_fit_maxiter is None else int(theta_fit_maxiter)
        self.theta_restarts = 2 if theta_restarts is None else int(theta_restarts)   # skopt's n_restarts_optimizer
        self._skopt_fit = None        # (told rows, told y, FitResult) of the last theta_fit="skopt" refit
        self.theta_refits = 0         # theta_fit="skopt" refits so far (diagnostics, tests)
        self.last_theta = None
        if candidate_backend not in ("torch", "numpy"):
            raise ValueError("candidate_backend must be 'torch' (sampled on the device) or 'numpy'")
        self.candidate_backend = candidate_backend
        self._tgen = None
        self._crng = None
        self.last_local_best = None
        self._seed = random_state
        self.Xi, self.yi = [], []
        self._Xt = np.empty((0, self.space.transformed_n_dims))   # transformed rows, one per told point
        self._engine = engine
        self.incremental = bool(incremental)   # False: refit on every ask, as skopt does
        # Sharded sweep (SURVEY.md §8(e)): every rank of the default process group holds the same optimizer (same tells, same
        # seed) and sweeps its own n_points/world candidates; one all-gather picks the winner, its owner broadcasts the row.
        # Opt-in (the SPMD server sets it): every rank must then make the same calls in the same order.
        self.shard = bool(shard) and self._world()[1] > 1
        if self.shard and random_state is None:
            import torch.distributed as dist
            box = [int(np.random.default_rng().integers(0, 2 ** 31))]
            dist.broadcast_object_list(box, src=0)          # ranks must draw the same initial points
            random_state = box[0]
            self._seed = random_state
            self.rng = np.random.default_rng(random_state)
        self._est_seed = None
        if theta_fit == "skopt":      # skopt cooks its GP once, with a seed drawn from the optimizer's random_state
            from .thetafit import estimator_seed
            self._est_seed = estimator_seed(random_state)
        self._fit_state = None        # (θ key, rows in the engine, digest of those rows): lets a request that only adds trials append
        self.last_fit = None          # "fit" | "append" | "reuse": what the last ask did to the engine (diagnostics, tests)
        self.last_best = None

    def close(self):
        """Release the GP or forest engine (its libkbo handle and device memory); a later ask makes a fresh one.  A GbrtEngine
        passed as base_estimator is the caller's and stays open."""
        if self._engine is not None and self._engine is not self._gbrt:
            self._engine.close()
            self._engine = None
        self._fit_state = None

    # ------------------------------------------------------------------------------------------------------
    def tell(self, x, y, xt=None):
        """``xt``: the rows already in the transformed space (the request scan computes them column-wise); must equal
        ``space.transform(x)``."""
        if len(x) and not isinstance(x[0], (list, tuple)):
            x, y = [x], [y]
            xt = None if xt is None else np.atleast_2d(xt)
        if len(x) != len(y):
            raise ValueError("x and y must have the same length")
        rows = [list(p) for p in x]
        self.Xi.extend(rows)
        self.yi.extend([float(v) for v in y])
        if rows:
            new = self.space.transform(rows) if xt is None else np.asarray(xt, dtype=np.float64).reshape(len(rows), -1)
            self._Xt = np.concatenate([self._Xt, new])

    def _get_engine(self, ls):
        from .gp import GPEngine
        kernel = "rbf" if self._hmap is not None else self.kernel
        if self._engine is None:
            self._engine = GPEngine(self.device, kernel=kernel, amplitude=self.amplitude, noise=self.noise,
                                    acq=self.acq, xi=self.xi, kappa=self.kappa, var_mode=self.var_mode)
        e = self._engine
        e.kernel, e.acq, e.amplitude, e.noise, e.xi, e.kappa = kernel, self.acq, self.amplitude, self.noise, self.xi, self.kappa
        self._set_length_scale(e, ls)
        return e

    def _set_length_scale(self, e, ls):
        """Every length scale the engine is fitted at passes here.  With kernel="hamming", ``ls`` are the Hamming weights l_j,
        mapped to the one-hot columns' RBF length scales, and "auto" sweeps at those θ take the path HammingMap.var_mode
        chooses."""
        if self._hmap is None:
            e.length_scale = np.atleast_1d(np.asarray(ls, dtype=np.float64))
            return
        e.length_scale = self._hmap.length_scale(ls)
        e.var_mode = self._hmap.var_mode(ls, self.var_mode)

    def _tell_engine(self, eng, Xt, ya, max_append=16):
        """Bring the engine to the history (Xt, ya) at its current θ.  Katib resends the whole history on every request and
        the constant liar extends it one row at a time, so most calls differ from what the engine already holds only past a
        long common prefix of rows: the engine keeps that prefix (kbo_fit_rebase — the leading blocks of L and L⁻¹ are the
        factors of the shorter history; targets are replaced wholesale, so a lie that became an observation costs nothing) and
        the few new rows are appended (kbo_fit_append, O(N²) each) while there is room in the last fit's row pitch (its N
        rounded up to 64, kept by a rebase: eng.room()).  Anything else —
        a different θ, an edited early row, many new rows — refits (O(N³)) as skopt does on every tell."""
        key = (eng.kernel, tuple(np.atleast_1d(eng.length_scale).tolist()), eng.amplitude, eng.noise, eng.normalize_y, eng.var_mode,
               eng.acq, eng.xi, eng.kappa)
        n, st = len(ya), self._fit_state
        self._fit_state = None          # stays None if anything below raises: the engine state is then unknown
        done = None
        if self.incremental and st is not None and st[0] == key and n >= 1:
            Xh, yh = st[1], st[2]
            m = min(n, len(yh))
            diff = np.flatnonzero((Xt[:m] != Xh[:m]).any(axis=1))
            p = int(diff[0]) if len(diff) else m          # rows [0, p) of the engine are rows [0, p) of the new history
            if p >= 1 and n - p <= max_append and p + eng.room() + (len(yh) - p) >= n:
                if p == n == len(yh) and np.array_equal(ya, yh):
                    done = "reuse"
                else:
                    if p != len(yh) or not np.array_equal(ya[:p], yh[:p]):   # rows dropped or targets changed
                        eng.rebase(p, ya[:p])
                    for i in range(p, n):
                        eng.append(Xt[i], ya[i])
                    done = "append" if n > p else "rebase"
        if done is None:
            eng.tell(Xt, ya)
            done = "fit"
        self.last_fit = done
        self._fit_state = (key, np.array(Xt, dtype=np.float64, copy=True), np.array(ya, dtype=np.float64, copy=True))

    @staticmethod
    def _world():
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                return dist.get_rank(), dist.get_world_size()
        except Exception:
            pass
        return 0, 1

    def _sweep(self, eng, cand, global_offset=0):
        try:
            return eng.ask(cand, global_offset=global_offset)
        except Exception:
            self._fit_state = None      # e.g. an appended row made K singular: the next ask must refit from the history
            raise

    def _default_ls(self):
        if self._hmap is not None:    # skopt's HammingKernel(length_scale=1.0) start
            return 1.0 if self.length_scale is None else self.length_scale
        return 0.3 * np.sqrt(self.space.transformed_n_dims) if self.length_scale is None else self.length_scale

    def _hedge_gains(self, eng, Xt, ya, lie):
        """The gains the draw of this ask uses, advanced where skopt's tell would advance them.  Nothing is stored here:
        _hedge_pick commits them together with the new picks once the sweep has succeeded, so an ask that fails cannot
        subtract the same picks twice."""
        if lie:
            prev, base = self._lie_next_xs, self._lie_gains
        else:
            h = self._hedge_hist
            changed = h is None or h[0].shape != Xt.shape or not (np.array_equal(h[0], Xt) and np.array_equal(h[1], ya))
            prev, base = (self.next_xs if changed else None), self.gains
        return base if prev is None else base - eng.predict_mean(prev)

    def _get_forest(self):
        """The RF / ET engine, made on first use with a seed fixed for its lifetime: the same history gives the same forest; or
        the GbrtEngine passed as base_estimator, set to this optimizer's acquisition."""
        if self._gbrt is not None:
            self._engine = g = self._gbrt
            g.acq, g.xi, g.kappa = self.acq, self.xi, self.kappa
            return g
        from .forest import ForestEngine
        if self._engine is None:
            seed = int(self._seed) if self._seed is not None else int(self.rng.integers(0, 2 ** 31))
            self._engine = ForestEngine(self.device, kind=self.base_estimator, seed=seed, acq=self.acq, xi=self.xi, kappa=self.kappa)
        return self._engine

    def _ask_one(self, X, y):
        if len(y) < max(self.n_initial_points, 1):
            self._last_gp = False
            return self.space.inverse_transform(self.space.rvs_transformed(1, self.rng, np.float64))[0]
        self._last_gp = True
        n_told = len(self._Xt)
        Xt = self._Xt
        if len(X) > n_told:          # constant-liar rows appended by ask(n_points=k)
            Xt = np.concatenate([Xt, self.space.transform(X[n_told:])])
        ya = np.asarray(y, dtype=np.float64)
        if self.forest:              # refit on a changed history (every lie included), as skopt's tell does; raw y, no θ
            eng = self._get_forest()
            eng.tell(Xt, ya)
            self.last_fit = eng.last_fit
            return self._pick(eng, Xt, ya, len(X) > n_told)
        base = np.atleast_1d(np.asarray(self._default_ls(), dtype=np.float64))
        eng = self._get_engine(base)
        if self.theta_grid > 1 or self.theta_search > 0:   # choose θ by the GPU log-marginal likelihood
            cands = [(float(m), self.noise) for m in (np.geomspace(0.25, 4.0, self.theta_grid) if self.theta_grid > 1 else [1.0])]
            if self.theta_search > 0:
                tr = np.random.default_rng(0 if self._seed is None else int(self._seed) + 17)
                cands += [(float(np.exp(tr.uniform(np.log(0.2), np.log(5.0)))), float(np.exp(tr.uniform(np.log(1e-6), np.log(1e-1)))))
                          for _ in range(self.theta_search)]
            best_lml, best_t = -np.inf, (1.0, self.noise)
            if hasattr(eng, "lml_batch"):
                # all candidates in a few calls: the factorisations of a batch run concurrently on the device (kbo_lml_batch) —
                # the chain of diagonal blocks of one hides behind the others' — instead of one full fit per θ
                gb = max(1, min(8, int(2 ** 31 // max(1, 8 * len(ya) * len(ya)))))      # ≤ 2 GiB of Gram matrices per batch
                for i in range(0, len(cands), gb):
                    part = cands[i:i + gb]
                    lmls = eng.lml_batch(Xt, ya, [dict(length_scale=base * m, noise=nz) for m, nz in part])
                    for (m, nz), lml in zip(part, lmls):
                        if np.isfinite(lml) and lml > best_lml:
                            best_lml, best_t = float(lml), (m, nz)
            else:
                self._fit_state = None
                for m, nz in cands:
                    eng.length_scale, eng.noise = base * m, nz
                    eng.tell(Xt, ya)
                    try:
                        lml = eng.fit_info()["lml"]
                    except Exception:   # not positive definite at this θ
                        continue
                    if lml > best_lml:
                        best_lml, best_t = lml, (m, nz)
            eng.length_scale, eng.noise = base * best_t[0], best_t[1]
            self.last_theta = dict(length_scale=eng.length_scale.copy(), noise=eng.noise, lml=best_lml)
        if self.theta_fit == "skopt":
            self._skopt_theta(eng, self._Xt, ya[:n_told])
        if self.theta_fit == "lbfgs":
            from scipy.optimize import minimize
            Dt = self.space.transformed_n_dims
            ls0 = np.broadcast_to(np.atleast_1d(eng.length_scale), (Dt,)).copy() if self.ard else np.atleast_1d(eng.length_scale)[:1].copy()
            x0 = np.concatenate([np.log(ls0), [np.log(max(eng.noise, 1e-8))]])
            bounds = [(np.log(1e-2), np.log(1e2))] * len(ls0) + [(np.log(1e-8), np.log(1.0))]

            self._fit_state = None

            def negative_lml(t):
                eng.length_scale, eng.noise = np.exp(t[:-1]), float(np.exp(t[-1]))
                eng.tell(Xt, ya)
                try:
                    lml, g = eng.lml_grad()            # g: (log amp, log noise, log ℓ…)
                except Exception:                       # not positive definite at this θ
                    return 1e25, np.zeros_like(t)
                return -lml, -np.concatenate([g[2:], g[1:2]])

            maxiter = 25 if self.theta_fit_maxiter is None else self.theta_fit_maxiter
            res = minimize(negative_lml, x0, jac=True, method="L-BFGS-B", bounds=bounds, options=dict(maxiter=maxiter))
            eng.length_scale, eng.noise = np.exp(res.x[:-1]), float(np.exp(res.x[-1]))
            self.last_theta = dict(length_scale=eng.length_scale.copy(), noise=eng.noise, lml=-float(res.fun), nfev=int(res.nfev))
        self._tell_engine(eng, Xt, ya)
        return self._pick(eng, Xt, ya, len(X) > n_told)

    def _skopt_theta(self, eng, Xt, yt):
        """θ as skopt fits it, on the told history (Xt, yt): refitted when that history changed since the last fit, else
        reused.  Leaves the engine at the winner's θ (its noise plus sklearn's alpha on the diagonal)."""
        from . import thetafit
        st = self._skopt_fit
        if st is None or st[0].shape != Xt.shape or not (np.array_equal(st[0], Xt) and np.array_equal(st[1], yt)):
            if self._hmap is None:
                res = thetafit.fit(thetafit.engine_batch_fn(eng, Xt, yt), Xt.shape[1], self._est_seed, self.theta_restarts,
                                   self.theta_fit_maxiter)
            else:
                from .hamming import LS_BOUNDS
                res = thetafit.fit(thetafit.engine_batch_fn(eng, Xt, yt, hamming=self._hmap), self._hmap.n_dims, self._est_seed,
                                   self.theta_restarts, self.theta_fit_maxiter, ls_bounds=LS_BOUNDS)
            self._skopt_fit = st = (np.array(Xt, dtype=np.float64, copy=True), np.array(yt, dtype=np.float64, copy=True), res)
            self.theta_refits += 1
        res = st[2]
        th = thetafit.theta_dict(res.theta)
        eng.amplitude, eng.noise = th["amplitude"], th["noise"]
        self._set_length_scale(eng, th["length_scale"])
        self.last_theta = dict(amplitude=th["amplitude"], length_scale=th["length_scale"].copy(), noise=float(np.exp(res.theta[-1])),
                               lml=res.lml, winner=res.winner, batch_calls=res.batch_calls,
                               starts=[dict(theta0=p.theta0.copy(), theta=p.theta.copy(), neg_lml=p.fun, nit=p.nit, nfev=p.nfev,
                                            status=p.status, message=p.message) for p in res.starts])

    def _pick(self, eng, Xt, ya, lie):
        """Sample the candidates (this rank's share when sharded), sweep them with the fitted engine, and return the point."""
        rank, world = self._world() if self.shard else (0, 1)
        from .dist import global_argmax, shard_rows
        if world > 1 and self.n_points < world:     # identical on every rank, before any collective: all raise together
            raise ValueError(f"n_points={self.n_points} must be >= the number of ranks ({world}) when the grid is sharded")
        lo, hi = shard_rows(self.n_points, rank, world)
        if self.candidate_backend == "torch":
            import torch
            dev = torch.device("cuda", self.device)
            if self._tgen is None:
                self._tgen = torch.Generator(device=dev)
                base = int(self._seed) if self._seed is not None else int(self.rng.integers(0, 2 ** 31))
                self._tgen.manual_seed(base + 1000003 * rank)
            cand = self.space.rvs_transformed_torch(hi - lo, self._tgen, dev)
        else:
            if self._crng is None:
                self._crng = self.rng if world == 1 else np.random.default_rng([int(self._seed), rank])
            cand = self.space.rvs_transformed(hi - lo, self._crng, np.float32)
        if self._hmap is not None:
            cand = self._hmap.candidates(cand)
        if self.hedge:
            return self._hedge_pick(eng, cand, lo, rank, world, lie, Xt, ya)
        failed = None
        try:
            best = self._sweep(eng, cand, lo)
        except Exception as e:  # noqa: BLE001
            if world == 1:
                raise
            best, failed = None, f"{type(e).__name__}: {e}"   # still join the exchange: every rank raises there, none hangs
        self.last_local_best = best
        li = best.index - lo if best is not None else 0
        if world > 1:
            import torch
            import torch.distributed as dist
            cdev = torch.device("cuda", self.device) if dist.get_backend() == "nccl" else torch.device("cpu")
            best = global_argmax(best, device=cdev, failed=failed)
            owner = next(r for r in range(world) if shard_rows(self.n_points, r, world)[0] <= best.index < shard_rows(self.n_points, r, world)[1])
            rowt = torch.zeros(self.space.transformed_n_dims, dtype=torch.float64, device=cdev)
            if rank == owner:
                li = best.index - lo
                src = cand[li] if isinstance(cand, torch.Tensor) else torch.from_numpy(np.asarray(cand[li]))
                rowt.copy_(src.to(torch.float64))
            dist.broadcast(rowt, src=owner)
            row = rowt.cpu().numpy()[None, :]
        elif self.candidate_backend == "torch":
            import torch
            row = cand[li:li + 1].to(torch.float64).cpu().numpy()
        else:
            row = cand[li:li + 1].astype(np.float64)
        self.last_best = best
        return self.space.inverse_transform(row)[0]

    def _hedge_pick(self, eng, cand, lo, rank, world, lie, Xt, ya):
        """One sweep for EI, LCB and PI over the candidate set, the draw among the three picks, and the picks kept for the next
        gains update.  Sharded: one all-gather for the three winners, one all-reduce that gives every rank all three rows."""
        from .dist import global_argmax, shard_rows
        failed = None
        try:
            gains = self._hedge_gains(eng, Xt, ya, lie)
            local = eng.ask_multi(cand, list(HEDGE_ACQS), global_offset=lo)
        except Exception as e:  # noqa: BLE001
            self._fit_state = None      # e.g. an appended row made K singular: the next ask must refit from the history
            if world == 1:
                raise
            local, failed = None, f"{type(e).__name__}: {e}"   # still join the exchange: every rank raises there, none hangs
        self.last_local_best = local
        Dt = self.space.transformed_n_dims
        if world > 1:
            import torch
            import torch.distributed as dist
            cdev = torch.device("cuda", self.device) if dist.get_backend() == "nccl" else torch.device("cpu")
            bests = global_argmax(local, device=cdev, failed=failed, n=len(HEDGE_ACQS))
            rows = torch.zeros((len(HEDGE_ACQS), Dt), dtype=torch.float64, device=cdev)
            hi = shard_rows(self.n_points, rank, world)[1]
            for j, b in enumerate(bests):   # each winner's owner fills its row; the sum hands every rank all three
                if lo <= b.index < hi:
                    src = cand[b.index - lo]
                    rows[j].copy_((src if isinstance(src, torch.Tensor) else torch.from_numpy(np.asarray(src))).to(torch.float64))
            dist.all_reduce(rows)
            picks = rows.cpu().numpy()
        else:
            bests = local
            li = [b.index - lo for b in bests]
            if self.candidate_backend == "torch":
                import torch
                picks = cand[torch.tensor(li, device=cand.device)].to(torch.float64).cpu().numpy()
            else:
                picks = np.asarray(cand[li], dtype=np.float64)
        logits = gains - np.max(gains)
        probs = np.exp(self.eta * logits)
        probs /= probs.sum()
        j = int(np.argmax(self.rng.multinomial(1, probs)))
        if lie:
            self._lie_gains, self._lie_next_xs = gains, picks
        else:
            self.gains, self.next_xs = gains, picks
            self._hedge_hist = (np.array(Xt, dtype=np.float64, copy=True), np.array(ya, dtype=np.float64, copy=True))
        self.last_hedge = (bests, probs, j)
        self.last_best = bests[j]
        return self.space.inverse_transform(picks[j:j + 1])[0]

    def ask(self, n_points=None):
        if n_points is None:
            return self._ask_one(self.Xi, self.yi)
        X, y, out = list(self.Xi), list(self.yi), []
        for i in range(int(n_points)):
            x = self._ask_one(X, y)
            if i == 0 and self.hedge:   # the lies work on a copy of the gains, starting from this step's picks
                self._lie_gains = self.gains.copy()
                self._lie_next_xs = self.next_xs if self._last_gp else None
            out.append(x)
            if y:                      # constant liar, "cl_min"
                X.append(x)
                y.append(min(y))
        return out
