"""FP64 NumPy restatement of skopt's GBRT surrogate of ``bayesianoptimization`` — the contract ``kubeflow_b200/csrc/gbrt.cu`` is
tested against.  Imported by tests and the golden generator only.

Sources.  $SK = scikit-learn 1.9.0 ``sklearn/``:
  * ``ensemble/_gb.py:554-555,745-746``, ``dummy.py:594-596``: the init is ``DummyRegressor(strategy="quantile")``,
    ``np.percentile(y, 100·α)`` with NumPy's linear method, no weights;
  * ``_loss/loss.py`` PinballLoss: the negative gradient is α where y >= raw and α − 1 where y < raw;
  * ``ensemble/_gb.py:481-502``: each stage fits ``DecisionTreeRegressor(criterion="squared_error", splitter="best",
    max_depth=3, min_samples_split=2, min_samples_leaf=1)`` to the negative gradient, X cast to float32;
  * ``ensemble/_gb.py:250-266``, ``_loss/loss.py:662-673``, ``utils/stats.py``: every leaf value is replaced by
    ``_weighted_percentile(y − raw, ones, 100·α)`` (the inverted-CDF rule): the k-th smallest residual fl(y − raw) of the leaf, k
    the first 0-based index with k + 1 >= t, t = fl(fl(fl(100·α) / 100)·n), bumped to the next double above 0 when it is 0;
  * ``ensemble/_gb.py:269``: ``raw += fl(0.1 · value[leaf])``, the product and the sum rounded separately; predictions add the
    same terms in stage order from the init;
  * ``tree/_partitioner.pyx:195-213``: no split between sorted neighbours with v[p+1] <= fl32(v[p] + 1e-7); threshold
    v[p]/2 + v[p+1]/2 in FP64, v[p] where that equals v[p+1] or is infinite; a float32 x goes left where x <= threshold.

skopt (not installed here; restated from memory and marked [RECALL]):
  * [RECALL] ``cook_estimator("GBRT")`` is ``GradientBoostingQuantileRegressor(quantiles=[0.16, 0.5, 0.84],
    base_estimator=GradientBoostingRegressor(n_estimators=30, loss="quantile"))``: three clones, one per α, fitted separately;
  * [RECALL] ``predict(return_std=True)``: mean = chain(0.5), std = (chain(0.84) − chain(0.16)) / 2, which is negative where the
    quantiles cross; EI and PI are 0 where std <= 0, LCB takes std as it is; y is raw (not normalised).

The split search is a counting problem.  Every gradient is α or α − 1 and every weight is 1, so with n samples in the node, nl / nr
going left / right, P of the n with y >= raw and pl / pr of those going left / right, sklearn's proxy sl²/nl + sr²/nr equals
pl²/nl + pr²/nr − 2·P·(1 − α) + n·(1 − α)², and the best split is the argmax of (pl²·nr + pr²·nl) / (nl·nr): integer counts,
compared exactly, the same for every α.  Two deliberate differences from sklearn, stated once:
  * an exact tie goes to the lowest feature, then the lowest position, where sklearn visits the features in a random order and
    lets FP64 rounding decide between exact ties;
  * a pure node (P ∈ {0, n}) is a leaf.  sklearn tests its FP64 impurity against DBL_EPSILON, and a pure node's impurity is
    rounding noise that can exceed it at α = 0.16 / 0.84 (sklearn then splits the node; the split changes no prediction only if
    every child keeps the same leaf value, which the replaced percentiles need not).
"""
from __future__ import annotations

import math

import numpy as np

from oracle.forest_oracle import acquisition  # noqa: F401  (re-exported for the tests)

SKOPT_ALPHAS = (0.16, 0.5, 0.84)
N_STAGES = 30
LEARNING_RATE = 0.1
MAX_DEPTH = 3
FEATURE_THRESHOLD = np.float32(1e-7)


def init_value(y, alpha: float) -> float:
    """DummyRegressor(strategy="quantile", quantile=α): np.percentile, linear method."""
    return float(np.percentile(np.asarray(y, np.float64), 100.0 * alpha))


def leaf_rank(n: int, alpha: float) -> int:
    """0-based rank of the residual _weighted_percentile(·, ones(n), 100·α) returns."""
    t = (100.0 * alpha) / 100.0 * float(n)
    if t == 0.0:
        t = math.nextafter(0.0, 1.0)
    return min(max(int(math.ceil(t)) - 1, 0), n - 1)


def leaf_value(resid, alpha: float) -> float:
    r = np.sort(np.asarray(resid, np.float64), kind="stable")
    return float(r[leaf_rank(len(r), alpha)])


def _threshold(a, b) -> float:
    a, b = float(a), float(b)
    th = a / 2.0 + b / 2.0
    if th == b or math.isinf(th):
        th = a
    return th


def split_candidates(Xn, pos):
    """Per feature with a valid split: (feature, sorted order, sorted values, valid positions p, nl, nr, pl, pr), the split
    after sorted position p.  ``Xn`` float32 rows of the node, ``pos`` its y >= raw bits; ties in value keep row order."""
    c, D = Xn.shape
    P = int(pos.sum())
    out = []
    for f in range(D):
        order = np.argsort(Xn[:, f], kind="stable")
        v = Xn[order, f]
        cum = np.cumsum(pos[order].astype(np.int64))
        p = np.flatnonzero(v[1:] > (v[:-1] + FEATURE_THRESHOLD).astype(np.float32))
        if len(p) == 0:
            continue
        nl = p + 1
        nr = c - nl
        pl = cum[p]
        pr = P - pl
        out.append((f, order, v, p, nl, nr, pl, pr))
    return out


def exact_argmax(Xn, pos):
    """The exact argmax set of (pl²·nr + pr²·nl) / (nl·nr) over every valid split, as (feature, p, threshold, left-mask) in
    (feature, position) order, or [] when the node has no valid split."""
    cands = split_candidates(Xn, pos)
    if not cands:
        return []
    # num < n³ and den < n² fit int64 for n <= 65536; a float pass narrows the field, Python ints decide exactly
    score = [(pl * pl * nr + pr * pr * nl) / (nl * nr) for f, order, v, p, nl, nr, pl, pr in cands]
    top = max(float(s.max()) for s in score)
    best, keep = None, []
    for (f, order, v, p, nl, nr, pl, pr), s in zip(cands, score):
        for j in np.flatnonzero(s >= top * (1.0 - 1e-9)):
            n_ = int(pl[j]) ** 2 * int(nr[j]) + int(pr[j]) ** 2 * int(nl[j])
            d_ = int(nl[j]) * int(nr[j])
            if best is None or n_ * best[1] > best[0] * d_:
                best, keep = (n_, d_), [(f, j, order, v, p)]
            elif n_ * best[1] == best[0] * d_:
                keep.append((f, j, order, v, p))
    res = []
    for f, j, order, v, p in keep:
        q = int(p[j])
        left = np.zeros(len(Xn), bool)
        left[order[:q + 1]] = True
        res.append((f, q, _threshold(v[q], v[q + 1]), left))
    return res


def build_tree(X32, y, raw, alpha: float):
    """One stage: the tree on the y >= raw bits, its leaves replaced by the residual percentile.  Returns (tree, leaf of every
    row).  ``tree`` in sklearn's ``tree_`` layout (depth-first preorder, left first): feature (-2 at leaves), threshold (-2 at
    leaves), left / right (-1 at leaves), value (the replaced value at leaves, the mean negative gradient elsewhere),
    n_node_samples, n_pos (rows with y >= raw), and ``tie``: the largest exact argmax set met at a node."""
    X32 = np.asarray(X32, np.float32)
    y, raw = np.asarray(y, np.float64), np.asarray(raw, np.float64)
    pos = y >= raw
    u = 1.0 - alpha
    rec = dict(feature=[], threshold=[], left=[], right=[], value=[], n_node_samples=[], n_pos=[])
    leaf_of = np.zeros(len(y), np.int64)
    tie = 0

    def grow(idx, depth):
        nonlocal tie
        k = len(rec["feature"])
        c, P = len(idx), int(pos[idx].sum())
        for key in rec:
            rec[key].append(0)
        rec["n_node_samples"][k], rec["n_pos"][k] = c, P
        split = []
        if depth < MAX_DEPTH and c >= 2 and 0 < P < c:
            split = exact_argmax(X32[idx], pos[idx])
            tie = max(tie, len(split))
        if not split:
            rec["feature"][k], rec["threshold"][k], rec["left"][k], rec["right"][k] = -2, -2.0, -1, -1
            rec["value"][k] = leaf_value(y[idx] - raw[idx], alpha)
            leaf_of[idx] = k
            return k
        f, _, th, left = split[0]
        rec["feature"][k], rec["threshold"][k] = f, th
        rec["value"][k] = (P * alpha - (c - P) * u) / c
        rec["left"][k] = grow(idx[left], depth + 1)
        rec["right"][k] = grow(idx[~left], depth + 1)
        return k

    grow(np.arange(len(y)), 0)
    tree = {k: np.asarray(v, dtype=np.float64 if k in ("threshold", "value") else np.int32) for k, v in rec.items()}
    tree["tie"] = tie
    return tree, leaf_of


def apply(tree, X):
    """Leaf id of each row (float32 x <= FP64 threshold goes left)."""
    X = np.asarray(X, np.float32)
    node = np.zeros(len(X), np.int64)
    while True:
        inner = tree["left"][node] >= 0
        if not inner.any():
            return node
        r = np.flatnonzero(inner)
        f = tree["feature"][node[r]]
        go = X[r, f].astype(np.float64) <= tree["threshold"][node[r]]
        node[r] = np.where(go, tree["left"][node[r]], tree["right"][node[r]])


def fit_chain(X, y, alpha: float, n_stages: int = N_STAGES):
    """One boosting chain: init, the stage trees, and raw after every stage (n_stages × N)."""
    X32 = np.asarray(X, np.float32)
    y = np.asarray(y, np.float64)
    init = init_value(y, alpha)
    raw = np.full(len(y), init)
    trees, raws = [], []
    for _ in range(n_stages):
        tree, leaf_of = build_tree(X32, y, raw, alpha)
        raw = raw + LEARNING_RATE * tree["value"][leaf_of]
        trees.append(tree)
        raws.append(raw.copy())
    return dict(alpha=alpha, init=init, trees=trees, raw=np.asarray(raws))


def predict_chain(chain, X):
    out = np.full(len(X), chain["init"])
    for tree in chain["trees"]:
        out = out + LEARNING_RATE * tree["value"][apply(tree, X)]
    return out


def fit(X, y, alphas=SKOPT_ALPHAS, n_stages: int = N_STAGES):
    return [fit_chain(X, y, a, n_stages) for a in alphas]


def predict(chains, X):
    """skopt's predict(return_std=True): (mu, std, the three chain predictions)."""
    q = np.asarray([predict_chain(c, X) for c in chains])
    return q[1], (q[2] - q[0]) / 2.0, q
