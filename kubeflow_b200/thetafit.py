"""skopt's hyper-parameter fit of the GP, with its starts run in lockstep.

skopt's default GP (``cook_estimator``) is ``ConstantKernel(1.0, (0.01, 1000)) * Matern(ν=2.5, ℓ=ones(D), bounds (0.01, 100))``
plus a ``WhiteKernel``, ``normalize_y=True``, ``n_restarts_optimizer=2``; sklearn's ``GaussianProcessRegressor.fit`` maximises
the log-marginal likelihood over θ = (log amp, log ℓ_1..D, log noise) by SciPy's L-BFGS-B from the kernel's own θ and from
``n_restarts_optimizer`` points drawn uniformly in the log bounds ($SK/_gpr.py:299-339), and keeps the best optimum.

Here the starts run side by side: one thread per ``scipy.optimize.minimize``, and an evaluator that sends the pending θ of every
live start to the device in one batched call (``GPEngine.lml_grad_batch``) once each live start has submitted a θ or finished.
A θ's (LML, gradient) does not depend on the batch it is computed in, so every start follows exactly the path it would follow
alone, and the result equals running the starts one after another.

Items marked [RECALL] restate skopt from memory (it is not a dependency of this package).
"""
from __future__ import annotations

import threading
from dataclasses import dataclass, field

import numpy as np

ALPHA = 1e-10                         # sklearn GaussianProcessRegressor's default alpha: added to the diagonal with the noise
AMP_BOUNDS = (0.01, 1000.0)           # ConstantKernel(1.0, (0.01, 1000.0)) in skopt's cook_estimator
LS_BOUNDS = (0.01, 100.0)             # Matern(length_scale_bounds=[(0.01, 100)] * n_dims)
NOISE_BOUNDS = (1e-5, 1e5)            # WhiteKernel's default noise_level_bounds [RECALL]


def bounds(n_dims: int, ls_bounds=LS_BOUNDS) -> np.ndarray:
    """(2 + n_dims, 2) log bounds in sklearn's θ order: log amp, log ℓ_1..n_dims, log noise.  ``ls_bounds``: the length scales'
    bounds (Matérn's by default; ``hamming.LS_BOUNDS`` for the HammingKernel's weights)."""
    rows = [AMP_BOUNDS] + [ls_bounds] * n_dims + [NOISE_BOUNDS]
    return np.log(np.asarray(rows, dtype=np.float64))


def estimator_seed(random_state) -> int:
    """The random_state skopt's Optimizer hands to cook_estimator: ``RandomState(random_state).randint(0, 2**31 - 1)``
    (``np.iinfo(np.int32).max``) [RECALL]."""
    return int(np.random.RandomState(random_state).randint(0, np.iinfo(np.int32).max))


def starts(n_dims: int, est_seed: int, n_restarts: int, ls_bounds=LS_BOUNDS) -> np.ndarray:
    """The initial θ of each L-BFGS-B run: the kernel's own θ = log(1, …, 1), then ``n_restarts`` draws of
    ``RandomState(est_seed).uniform(lo, hi)``, in order, as sklearn's fit draws them (it re-seeds on every fit, so a refit
    starts from the same points)."""
    b = bounds(n_dims, ls_bounds)
    rng = np.random.RandomState(est_seed)
    return np.stack([np.zeros(len(b))] + [rng.uniform(b[:, 0], b[:, 1]) for _ in range(n_restarts)])


def theta_dict(t) -> dict:
    """Engine θ of a θ vector in sklearn's order; the device's diagonal term is noise + sklearn's alpha."""
    t = np.asarray(t, dtype=np.float64)
    return dict(amplitude=float(np.exp(t[0])), length_scale=np.exp(t[1:-1]), noise=float(np.exp(t[-1])) + ALPHA)


def to_objective(lml: float, grad, noise: float):
    """(−LML, −∂LML/∂θ in sklearn's order) from the device's (LML, gradient in (log amp, log noise, log ℓ…) order).  The
    device differentiates with respect to log(noise + alpha); sklearn's ∂/∂log noise is that times noise / (noise + alpha).
    A θ whose Gram matrix is not positive definite is (+inf, 0), as sklearn's LML returns (−inf, 0) there."""
    grad = np.asarray(grad, dtype=np.float64)
    if not np.isfinite(lml):
        return np.inf, np.zeros(len(grad))
    g = np.concatenate([[grad[0]], grad[2:], [grad[1] * (noise / (noise + ALPHA))]])
    return -float(lml), -g


class Lockstep:
    """Runs one objective per start in its own thread and batches their evaluations: ``batch_fn(list of θ) -> list of
    (f, g)`` is called (from whichever thread completes the round) when every live start has a θ pending.  Rounds submit the
    θ in start order."""

    def __init__(self, n: int, batch_fn):
        self._cv = threading.Condition()
        self._batch_fn = batch_fn
        self._pending, self._results = {}, {}
        self._live = set(range(n))
        self.error = None
        self.calls = 0

    def evaluate(self, i: int, theta):
        with self._cv:
            self._pending[i] = np.array(theta, dtype=np.float64, copy=True)
            self._launch_if_ready()
            while i not in self._results and self.error is None:
                self._cv.wait()
            if i not in self._results:
                raise RuntimeError("a batched θ evaluation failed") from self.error
            return self._results.pop(i)

    def finish(self, i: int):
        with self._cv:
            self._live.discard(i)
            self._launch_if_ready()

    def fail(self, i: int, error: BaseException):
        with self._cv:
            self._live.discard(i)
            if self.error is None:
                self.error = error
            self._cv.notify_all()

    def _launch_if_ready(self):
        if self.error is not None or not self._pending or set(self._pending) != self._live:
            return
        idx = sorted(self._pending)
        thetas = [self._pending.pop(j) for j in idx]
        try:
            out = self._batch_fn(thetas)
        except BaseException as e:  # noqa: BLE001  every waiting start re-raises it
            self.error = e
            self._cv.notify_all()
            return
        self.calls += 1
        for j, r in zip(idx, out):
            self._results[j] = r
        self._cv.notify_all()


@dataclass
class StartResult:
    theta0: np.ndarray        # initial θ (sklearn order, logs)
    theta: np.ndarray         # final θ
    fun: float                # −LML at theta
    nit: int
    nfev: int
    status: int               # SciPy's L-BFGS-B status (0: converged, 1: iteration / evaluation limit, 2: abnormal)
    message: str


@dataclass
class FitResult:
    theta: np.ndarray         # the winner's θ (sklearn order, logs)
    lml: float                # its log-marginal likelihood
    winner: int               # index of the winning start (np.argmin of −LML: first on ties)
    starts: list = field(default_factory=list)   # StartResult per start
    batch_calls: int = 0      # batched device calls the lockstep made


def _minimize(fun, x0, b, maxiter):
    from scipy.optimize import minimize
    options = {} if maxiter is None else dict(maxiter=int(maxiter))
    return minimize(fun, x0, method="L-BFGS-B", jac=True, bounds=b, options=options)


def fit(batch_fn, n_dims: int, est_seed: int, n_restarts: int = 2, maxiter: int | None = None, lockstep: bool = True,
        ls_bounds=LS_BOUNDS) -> FitResult:
    """sklearn's restart search over skopt's bounds.  ``batch_fn(list of θ) -> list of (−LML, −gradient)`` in sklearn's order
    (see ``to_objective``).  ``lockstep=False`` runs the starts one after another, one θ per call (the reference the lockstep
    must equal).  ``maxiter``: L-BFGS-B's iteration limit (None: SciPy's default)."""
    x0s = starts(n_dims, est_seed, n_restarts, ls_bounds)
    b = bounds(n_dims, ls_bounds)
    res = [None] * len(x0s)
    calls = 0
    if lockstep:
        box = Lockstep(len(x0s), batch_fn)

        def run(i):
            try:
                res[i] = _minimize(lambda t: box.evaluate(i, t), x0s[i], b, maxiter)
            except BaseException as e:  # noqa: BLE001  the first error is re-raised below, after every start has stopped
                box.fail(i, e)
                return
            box.finish(i)

        threads = [threading.Thread(target=run, args=(i,), name=f"theta-start-{i}") for i in range(len(x0s))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if box.error is not None:
            raise box.error
        calls = box.calls
    else:
        def single(t):
            nonlocal calls
            calls += 1
            return batch_fn([np.array(t, dtype=np.float64, copy=True)])[0]
        for i, x0 in enumerate(x0s):
            res[i] = _minimize(single, x0, b, maxiter)
    per = [StartResult(theta0=x0s[i], theta=np.asarray(r.x, dtype=np.float64), fun=float(r.fun), nit=int(r.nit), nfev=int(r.nfev),
                       status=int(r.status), message=str(r.message)) for i, r in enumerate(res)]
    w = int(np.argmin([p.fun for p in per]))
    return FitResult(theta=per[w].theta, lml=-per[w].fun, winner=w, starts=per, batch_calls=calls)


def engine_batch_fn(eng, X, y, scratch_limit: int | None = None, hamming=None):
    """``batch_fn`` over a GPEngine: one ``lml_grad_batch`` per round, split into calls of as many θ as the engine's scratch
    limit holds (a θ's result does not depend on the split).  ``hamming``: a ``hamming.HammingMap``; θ's length scales are then
    the Hamming weights l_j, evaluated as RBF length scales of the one-hot columns, and the gradient is returned per l_j."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    y = np.ascontiguousarray(y, dtype=np.float64).reshape(-1)
    N, D = X.shape
    limit = eng.scratch_limit if scratch_limit is None else int(scratch_limit)
    per_call = max(1, min(64, limit // eng.lml_grad_lane_bytes(N, D, D)))

    def batch_fn(thetas):
        out = []
        for i in range(0, len(thetas), per_call):
            part = thetas[i:i + per_call]
            ths = [theta_dict(t) for t in part]
            if hamming is not None:
                for th in ths:
                    th["length_scale"] = hamming.length_scale(th["length_scale"])
            lml, grad = eng.lml_grad_batch(X, y, ths)
            if hamming is not None:
                grad = [np.concatenate([g[:2], hamming.grad(g[2:])]) for g in grad]
            out += [to_objective(v, g, float(np.exp(t[-1]))) for v, g, t in zip(lml, grad, part)]
        return out
    return batch_fn
