"""Writes tests/golden/forest_*.npz: RF trees fitted by the real scikit-learn (1.9.0) on imposed bootstrap counts, for
tests/test_forest_oracle.py (the restatement) and tests/test_gpu_forest.py (the device).  Run from the repository root:
``python -m oracle.make_golden_forest``.

Each case holds X (float32, the transformed [0, 1] coordinates), y, the Philox bootstrap counts of oracle.forest_oracle (T × N),
candidates Xc, per tree sklearn's ``tree_`` arrays (depth-first ids, as sklearn numbers them), and mu / sigma by skopt's
``_return_std`` over those trees.  sklearn visits features in a random order and accumulates its sums in its own order, so a
tree whose best and second-best split proxies at some node lie within 1e-9 (relative) of each other could legitimately differ
from the restatement; such a tree's counts are redrawn (seed + 1000·attempt) until no node is that close, and the trees must then
match exactly."""
from __future__ import annotations

import os

import numpy as np
from sklearn.tree import DecisionTreeRegressor

from oracle import forest_oracle as F

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden")

# (name, N, D, T, M, y kind); a few trees at the larger shapes, whole small forests at the small ones
CASES = [("forest_rf_n24_d2", 24, 2, 8, 64, "smooth"), ("forest_rf_n60_d3", 60, 3, 6, 128, "smooth"),
         ("forest_rf_n40_d4_grid", 40, 4, 5, 96, "grid"), ("forest_rf_n300_d6", 300, 6, 3, 256, "smooth")]


def _data(rng, N, D, ykind):
    X = rng.random((N, D)).astype(np.float32)
    if ykind == "grid":          # integer / one-hot style columns: many tied values per feature
        X[:, 0] = rng.integers(0, 5, N) / 4.0
        X[:, 1] = rng.integers(0, 2, N)
    y = np.sin(3.0 * X[:, 0]) + X[:, 1 % D] ** 2 + 0.3 * rng.standard_normal(N)
    return X, y.astype(np.float64)


def main():
    for ci, (name, N, D, T, M, ykind) in enumerate(CASES):
        rng = np.random.default_rng(100 + ci)
        X, y = _data(rng, N, D, ykind)
        counts = np.zeros((T, N), np.int32)
        trees, seeds = [], []
        for t in range(T):
            for attempt in range(2000):
                seed = 7 + ci + 1000 * attempt
                c = F.bootstrap_counts(N, t + 1, seed)[t]
                ref = F.build_tree(X, y, c, min_samples_leaf=3, kind="RF")
                if ref["near_tie"] > 1e-9:
                    break
            else:
                raise RuntimeError(f"{name}: no tie-free bootstrap for tree {t}")
            est = DecisionTreeRegressor(min_samples_leaf=3, random_state=t).fit(X, y, sample_weight=c.astype(np.float64))
            tr = est.tree_
            trees.append(dict(feature=tr.feature.astype(np.int32), threshold=tr.threshold.copy(), left=tr.children_left.astype(np.int32),
                              right=tr.children_right.astype(np.int32), value=tr.value[:, 0, 0].copy(), impurity=tr.impurity.copy(),
                              n_node_samples=tr.n_node_samples.astype(np.int32), weighted_n_node_samples=tr.weighted_n_node_samples.copy()))
            counts[t] = c
            seeds.append(seed)
        Xc = rng.random((M, D)).astype(np.float32)
        Xc[: M // 4] = X[rng.integers(0, N, M // 4)]            # candidates on training points: exactly at split neighbours
        mu, sd = F.predict(trees, Xc)
        arrays = dict(X=X, y=y, counts=counts, Xc=Xc, mu=mu, sigma=sd, seeds=np.asarray(seeds), n_trees=np.int32(T))
        for t, tr in enumerate(trees):
            for k, v in tr.items():
                arrays[f"t{t}_{k}"] = v
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrays)
        print(name, "trees", T, "nodes", [len(tr["feature"]) for tr in trees])


if __name__ == "__main__":
    main()
