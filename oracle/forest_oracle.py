"""FP64 NumPy restatement of the forest surrogates of ``bayesianoptimization`` with ``base_estimator`` RF / ET — the contract
``kubeflow_b200/csrc/forest.cu`` is tested against.  Imported by tests only.

Sources.  $SKT = scikit-learn 1.9.0 ``sklearn/tree`` (its ``.pyx`` sources ship with the wheel):
  * ``_tree.pyx:230-251``      a node is a leaf if it holds < 2·min_samples_leaf samples or its impurity is <= DBL_EPSILON;
  * ``_criterion.pyx:938-940`` MSE impurity  Σ(w·y)·y / Σw − (Σw·y / Σw)²;  node value Σw·y / Σw;
  * ``_criterion.pyx:944-973`` split proxy   sum_l² / w_l + sum_r² / w_r, sum_r = sum_total − sum_l;
  * ``_partitioner.pyx:195-213`` and ``_partitioner.pxd:13``: no split between sorted neighbours with v[p+1] <= v[p] + 1e-7, the
    sum taken in float32 (FEATURE_THRESHOLD is a float32_t);
  * ``_splitter.pyx:~420-470`` best splitter: both sides keep min_samples_leaf samples (counted as distinct samples, not
    weight), a later candidate replaces the best only if its proxy is strictly greater, threshold v[p]/2.0 + v[p+1]/2.0 in FP64,
    v[p] where that equals v[p+1] or is infinite;
  * ``_splitter.pyx:590-665`` random splitter: min / max over the node (float32), the feature is constant if
    max <= min + 1e-7 (float32), threshold uniform in [min, max), min where it equals max, then the same side and proxy rules;
  * prediction: ``x <= threshold`` goes left, float32 x against the FP64 threshold.

skopt (not installed here; restated from memory and marked [RECALL]):
  * [RECALL] ``skopt.utils.cook_estimator``: "RF" → ``RandomForestRegressor(n_estimators=100, min_samples_leaf=3)``, "ET" →
    ``ExtraTreesRegressor(n_estimators=100, min_samples_leaf=3)``; ``min_variance = 0``; every feature at every node.
  * [RECALL] sklearn's forest fits tree t on the bootstrap draws as sample weights (the draw counts); ET does not bootstrap.
  * [RECALL] ``skopt.learning.forest._return_std``: per tree, var = impurity at the leaf (values below min_variance raised to it),
    std += var + value²; std /= T; std −= mean²; negatives to 0; std = std ** 0.5.  The mean is the forest's mean prediction.
  * [RECALL] ``skopt.Optimizer``: y is not normalised for tree estimators; EI / PI / LCB on the raw mean and std, EI and PI 0 where
    std = 0; ``acq_optimizer="lbfgs"`` with a tree estimator is an error ("The regressor ... should run with
    acq_optimizer='sampling'.").

Here, as on the device: ties across features go to the lowest feature index (sklearn visits features in a random order), the
mean and second moment are summed in tree order, and the random draws are Philox4x32-10 (``bootstrap_counts``, ``et_uniform``)
instead of NumPy's RandomState."""
from __future__ import annotations

import math

import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps
FEATURE_THRESHOLD = np.float32(1e-7)
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, seed):
    """Philox4x32-10 (Salmon et al., SC'11) on uint64 arrays holding 32-bit words; key = (seed low, seed high)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M32 for c in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint64(int(seed) & 0xFFFFFFFF), np.uint64((int(seed) >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def bootstrap_counts(N: int, T: int, seed: int) -> np.ndarray:
    """T × N draw counts: draw d of tree t is sample (u32·N) >> 32, u32 = word 0 of Philox counter (d, t, 0, 0)."""
    d = np.arange(N, dtype=np.uint64)[None, :]
    t = np.arange(T, dtype=np.uint64)[:, None]
    w0 = philox4x32_10(d, t, 0, 0, seed)[0]
    idx = ((w0 * np.uint64(N)) >> np.uint64(32)).astype(np.int64)
    out = np.zeros((T, N), np.int32)
    for k in range(T):
        out[k] = np.bincount(idx[k], minlength=N)
    return out


def et_uniform(seed: int, tree: int, node, feature) -> np.ndarray:
    """The 53-bit uniform of words 0 and 1 of Philox counter (node, tree, feature, 1): NumPy's (a >> 5, b >> 6) construction."""
    w = philox4x32_10(node, tree, feature, 1, seed)
    return ((w[0] >> np.uint64(5)).astype(np.float64) * 67108864.0 + (w[1] >> np.uint64(6)).astype(np.float64)) / 9007199254740992.0


def et_threshold(u, mn, mx):
    """(max − min)·u + min in FP64 from float32 min / max; min where it equals max ($SKT/_splitter.pyx:633-654)."""
    lo, hi = np.asarray(mn, np.float64), np.asarray(mx, np.float64)
    with np.errstate(invalid="ignore"):          # rows without samples (min +inf, max -inf) come out NaN
        th = (hi - lo) * u + lo
    return np.where(th == hi, lo, th)


def _stats(y, w):
    wy = w * y
    sw, swy, swyy = float(np.sum(w)), float(np.sum(wy)), float(np.sum(wy * y))
    value = swy / sw
    return sw, swy, value, swyy / sw - value * value      # Cython's (x / w)**2.0 compiles to x·x, not pow()


def _best_split(Xn, yn, wn, sw, swy, msl):
    """Best splitter over every feature.  Returns (proxy, feature, threshold, left mask) or None, and the second-best proxy."""
    c, D = Xn.shape
    order = np.argsort(Xn, axis=0, kind="stable")
    V = np.take_along_axis(Xn, order, 0)
    cw = np.cumsum(wn[order], axis=0)
    cwy = np.cumsum((wn * yn)[order], axis=0)
    nl = np.arange(1, c + 1)[:-1, None]
    valid = (V[1:] > V[:-1] + FEATURE_THRESHOLD) & (nl >= msl) & (c - nl >= msl)
    wl, sl = cw[:-1], cwy[:-1]
    with np.errstate(divide="ignore", invalid="ignore"):
        wr, sr = sw - wl, swy - sl
        proxy = np.where(valid, sl * sl / wl + sr * sr / wr, -np.inf)
    if not valid.any():
        return None, -np.inf
    per_f = proxy.max(axis=0)
    f = int(np.argmax(per_f))
    p = int(np.argmax(proxy[:, f]))
    a, b = np.float64(V[p, f]), np.float64(V[p + 1, f])
    th = a / 2.0 + b / 2.0
    if th == b or math.isinf(th):
        th = a
    left = np.zeros(c, bool)
    left[order[:p + 1, f]] = True
    flat = np.sort(proxy[valid])
    second = flat[-2] if len(flat) > 1 else -np.inf
    return (float(proxy[p, f]), f, float(th), left), float(second)


def _random_split(Xn, yn, wn, sw, swy, msl, draw):
    """Random splitter: draw(feature, min, max) gives the threshold of each non-constant feature."""
    c, D = Xn.shape
    best, second = None, -np.inf
    for f in range(D):
        col = Xn[:, f]
        mn, mx = col.min(), col.max()
        if mx <= np.float32(mn + FEATURE_THRESHOLD):
            continue
        th = float(draw(f, mn, mx))
        left = col.astype(np.float64) <= th
        n_left = int(left.sum())
        if n_left < msl or c - n_left < msl:
            continue
        wl, sl = float(np.sum(wn[left])), float(np.sum((wn * yn)[left]))
        wr, sr = sw - wl, swy - sl
        proxy = sl * sl / wl + sr * sr / wr
        if best is None or proxy > best[0]:
            if best is not None:
                second = max(second, best[0])
            best = (proxy, f, th, left)
        else:
            second = max(second, proxy)
    return best, second


def build_tree(X, y, w=None, *, min_samples_leaf=3, kind="RF", draws=None):
    """One tree, nodes numbered breadth-first.  X is cast to float32; w: sample weights (bootstrap counts; samples of weight 0
    are left out, as sklearn does).  ET: ``draws(node, feature, min, max)`` gives each threshold.  Returns sklearn's ``tree_``
    arrays plus ``near_tie``: the smallest relative gap between a node's best and second-best proxy."""
    X = np.asarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.float64)
    w = np.ones(len(y)) if w is None else np.asarray(w, dtype=np.float64)
    nodes = [np.flatnonzero(w > 0)]
    rec = dict(feature=[], threshold=[], left=[], right=[], value=[], impurity=[], n_node_samples=[], weighted_n_node_samples=[])
    near = np.inf
    k = 0
    while k < len(nodes):
        idx = nodes[k]
        c = len(idx)
        sw, swy, value, imp = _stats(y[idx], w[idx])
        for key, v in (("value", value), ("impurity", imp), ("n_node_samples", c), ("weighted_n_node_samples", sw)):
            rec[key].append(v)
        split = None
        if not (c < 2 * min_samples_leaf or imp <= DBL_EPSILON):
            if kind == "RF":
                split, second = _best_split(X[idx], y[idx], w[idx], sw, swy, min_samples_leaf)
            else:
                split, second = _random_split(X[idx], y[idx], w[idx], sw, swy, min_samples_leaf, lambda f, a, b, _k=k: draws(_k, f, a, b))
            if split is not None and np.isfinite(second):
                near = min(near, (split[0] - second) / abs(split[0]))
        if split is None:
            rec["feature"].append(-2)
            rec["threshold"].append(-2.0)
            rec["left"].append(-1)
            rec["right"].append(-1)
        else:
            _, f, th, left = split
            rec["feature"].append(f)
            rec["threshold"].append(th)
            rec["left"].append(len(nodes))
            rec["right"].append(len(nodes) + 1)
            nodes += [idx[left], idx[~left]]
        k += 1
    out = {key: np.asarray(v, dtype=np.int32 if key in ("feature", "left", "right", "n_node_samples") else np.float64) for key, v in rec.items()}
    out["near_tie"] = near
    return out


def build_forest(X, y, *, kind="RF", n_trees=100, min_samples_leaf=3, seed=0, counts=None):
    """The forest the device builds: RF on Philox bootstrap counts (or ``counts``), ET on Philox thresholds."""
    X = np.asarray(X, dtype=np.float32)
    trees = []
    if kind == "RF":
        counts = bootstrap_counts(len(y), n_trees, seed) if counts is None else counts
        for t in range(n_trees):
            trees.append(build_tree(X, y, counts[t], min_samples_leaf=min_samples_leaf, kind="RF"))
    else:
        for t in range(n_trees):
            draws = lambda k, f, a, b, _t=t: et_threshold(et_uniform(seed, _t, k, f), a, b)
            trees.append(build_tree(X, y, None, min_samples_leaf=min_samples_leaf, kind="ET", draws=draws))
    return trees


def apply(tree, X):
    """Leaf id of each row (float32 x <= FP64 threshold goes left)."""
    X = np.asarray(X, dtype=np.float32)
    node = np.zeros(len(X), np.int64)
    while True:
        inner = tree["left"][node] >= 0
        if not inner.any():
            return node
        r = np.flatnonzero(inner)
        f = tree["feature"][node[r]]
        go_left = X[r, f].astype(np.float64) <= tree["threshold"][node[r]]
        node[r] = np.where(go_left, tree["left"][node[r]], tree["right"][node[r]])


def predict(trees, X, min_variance=0.0):
    """skopt's forest predict(return_std=True), summed in tree order: (mu, std)."""
    mu = np.zeros(len(X))
    second = np.zeros(len(X))
    for tree in trees:
        leaf = apply(tree, X)
        v = tree["value"][leaf]
        var = tree["impurity"][leaf].copy()
        var[var < min_variance] = min_variance
        mu += v
        second += var + v ** 2
    mu /= len(trees)
    second /= len(trees)
    second -= mu ** 2.0
    second[second < 0.0] = 0.0
    return mu, np.sqrt(second)


def acquisition(kind, mu, std, y_opt, xi=0.01, kappa=1.96):
    """EI / PI (0 where std <= 0) and LCB as a value to maximise, -(mu - kappa·std) with std as it is (GBRT's may be negative):
    skopt.acquisition.gaussian_*."""
    mu, std = np.asarray(mu, np.float64), np.asarray(std, np.float64)
    if kind == "lcb":
        return -(mu - kappa * std)
    out = np.zeros_like(mu)
    m = std > 0
    imp = y_opt - xi - mu[m]
    z = imp / std[m]
    cdf = 0.5 * np.array([math.erfc(-v / math.sqrt(2.0)) for v in z])
    if kind == "pi":
        out[m] = cdf
    else:
        out[m] = imp * cdf + std[m] * np.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    return out
