"""CPU: the GBRT restatement oracle/gbrt_oracle.py against scikit-learn 1.9.0's quantile GradientBoostingRegressor chains in
tests/golden/gbrt_*.npz (oracle/make_golden_gbrt.py).

* Replay: on sklearn's own trees, sklearn's split at every node lies in the restatement's exact argmax set, and the restatement's
  init, leaf values, raw after every stage and probe predictions equal sklearn's bit for bit.  The one allowed exception is a
  pure node sklearn split (its FP64 impurity is rounding noise above DBL_EPSILON), counted, and only at α not exact in binary.
* Free run: where the generator found no exact tie (D = 1, α exact in binary), the restatement's own chain is sklearn's.
* Percentiles: the init is np.percentile's linear rule, and the leaf rank is _weighted_percentile's inverted-CDF rule."""
import glob
import os

import numpy as np
import pytest

from oracle import gbrt_oracle as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(glob.glob(os.path.join(GOLDEN, "gbrt_*.npz")))
EXACT = (0.25, 0.5, 0.75)


def _tree(z, c, s):
    return {k: z[f"c{c}_s{s}_{k}"] for k in ("feature", "threshold", "left", "right", "value", "n_node_samples")}


def _members(tree, X):
    """Rows reaching each node of a tree in sklearn's layout."""
    out, stack = {}, [(0, np.arange(len(X)))]
    while stack:
        k, r = stack.pop()
        out[k] = r
        if tree["left"][k] >= 0:
            go = X[r, tree["feature"][k]].astype(np.float64) <= tree["threshold"][k]
            stack += [(int(tree["left"][k]), r[go]), (int(tree["right"][k]), r[~go])]
    return out


@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[5:-4])
def test_replay_of_sklearns_trees(path):
    z = np.load(path)
    X32, y = z["X"].astype(np.float32), z["y"]
    pure_splits = 0
    for c, a in enumerate(z["alphas"]):
        a = float(a)
        init = G.init_value(y, a)
        assert init == float(z[f"c{c}_init"])
        raw = np.full(len(y), init)
        chain = dict(init=init, trees=[])
        for s in range(G.N_STAGES):
            t = _tree(z, c, s)
            pos = y >= raw
            for k, r in _members(t, X32).items():
                if t["left"][k] < 0:
                    assert G.leaf_value(y[r] - raw[r], a) == t["value"][k], f"c{c} s{s} leaf {k}"
                    continue
                if pos[r].all() or not pos[r].any():
                    pure_splits += 1
                    assert a not in EXACT, f"c{c} s{s} node {k}: sklearn split a pure node at α = {a}"
                    continue
                best = G.exact_argmax(X32[r], pos[r])
                assert any(f == t["feature"][k] and th == t["threshold"][k] for f, _, th, _ in best), f"c{c} s{s} node {k}"
            leaf = G.apply(t, X32)
            raw = raw + G.LEARNING_RATE * t["value"][leaf]
            assert np.array_equal(raw, z[f"c{c}_raw"][s]), f"c{c} s{s}: raw"
            chain["trees"].append(t)
        assert np.array_equal(G.predict_chain(chain, z["Xc"]), z[f"c{c}_pred"])
    print(f"{os.path.basename(path)}: {pure_splits} pure nodes split by sklearn")


@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[5:-4])
def test_free_run_equals_sklearn_where_no_tie_was_met(path):
    z = np.load(path)
    free = [c for c in range(3) if int(z[f"c{c}_free"])]
    if not free:
        pytest.skip("no chain of this case is free of exact ties")
    for c in free:
        own = G.fit_chain(z["X"], z["y"], float(z["alphas"][c]))
        for s in range(G.N_STAGES):
            t = _tree(z, c, s)
            for k in ("feature", "threshold", "left", "right", "n_node_samples"):
                assert np.array_equal(own["trees"][s][k], t[k]), f"c{c} s{s} {k}"
            leaves = t["left"] < 0
            assert np.array_equal(own["trees"][s]["value"][leaves], t["value"][leaves]), f"c{c} s{s} leaf values"
        assert np.array_equal(own["raw"], z[f"c{c}_raw"])
        assert np.array_equal(G.predict_chain(own, z["Xc"]), z[f"c{c}_pred"])


def test_some_golden_chain_runs_free():
    assert any(int(np.load(p)[f"c{c}_free"]) for p in CASES for c in range(3))


@pytest.mark.parametrize("alpha", [0.16, 0.25, 0.5, 0.75, 0.84])
def test_init_is_the_linear_percentile(alpha):
    rng = np.random.default_rng(int(alpha * 100))
    for n in (1, 2, 3, 7, 100, 1001):
        y = np.round(rng.standard_normal(n) * 8) / 8
        ys = np.sort(y)
        v = (n - 1) * ((100.0 * alpha) / 100.0)
        i = int(np.floor(v))
        if v >= n - 1:
            ref = ys[-1]
        else:
            g = v - i
            d = ys[i + 1] - ys[i]
            ref = ys[i + 1] - d * (1 - g) if g >= 0.5 else ys[i] + d * g
        assert G.init_value(y, alpha) == ref          # the rule gbrt.cu's init kernel states


@pytest.mark.parametrize("alpha", [0.16, 0.25, 0.5, 0.75, 0.84])
def test_leaf_rank_is_the_inverted_cdf_rule(alpha):
    sk = pytest.importorskip("sklearn.utils.stats")
    for n in range(1, 400):
        r = np.arange(n, dtype=np.float64)
        assert G.leaf_rank(n, alpha) == int(sk._weighted_percentile(r, np.ones(n), 100 * alpha)), n
