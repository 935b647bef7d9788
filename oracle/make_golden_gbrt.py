"""Generate tests/golden/gbrt_*.npz: scikit-learn 1.9.0's GradientBoostingRegressor(loss="quantile", n_estimators=30), the
chain skopt's GBRT surrogate is made of, fitted at skopt's α (0.16, 0.5, 0.84) and at α that are exact in binary (0.25, 0.5,
0.75), with every stage's tree, raw after every stage and the predictions at probe rows.  Run from the repository root:
``python -m oracle.make_golden_gbrt``.

Per case: X (N × D), y, Xc (probe rows), alphas (3), and per chain c: c{c}_init, c{c}_raw (stages × N), c{c}_pred (probe
predictions), c{c}_free (1 where D = 1, α is exact in binary and the restatement met no exact tie in its own run: its whole
chain must then equal sklearn's), and per stage s the tree_ arrays c{c}_s{s}_{feature, threshold, left, right, value,
n_node_samples}."""
from __future__ import annotations

import os

import numpy as np

from oracle import gbrt_oracle as G

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SKOPT = G.SKOPT_ALPHAS
EXACT = (0.25, 0.5, 0.75)


def case(seed, N, D, *, grid_cols=(), tied_y=False):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    for f in grid_cols:                      # integer-like columns with many equal values
        X[:, f] = np.floor(X[:, f] * 6) / 5
    y = np.sin(3 * X).sum(1) + 0.3 * rng.standard_normal(N)
    if tied_y:
        y = np.round(y * 4) / 4
    Xc = np.concatenate([rng.random((64, D)), X[:16]])
    return X, y, Xc


CASES = {
    "n24_d1_exact": (case(1, 24, 1), EXACT),
    "n60_d1_grid_exact": (case(2, 60, 1, grid_cols=(0,), tied_y=True), EXACT),
    "n200_d1_skopt": (case(3, 200, 1), SKOPT),
    "n100_d3_grid_skopt": (case(4, 100, 3, grid_cols=(0, 2)), SKOPT),
    "n200_d4_skopt": (case(5, 200, 4, grid_cols=(1,), tied_y=True), SKOPT),
    "n150_d2_exact": (case(6, 150, 2, grid_cols=(0,)), EXACT),
}


def main():
    from sklearn.ensemble import GradientBoostingRegressor
    os.makedirs(OUT, exist_ok=True)
    for name, ((X, y, Xc), alphas) in CASES.items():
        z = dict(X=X, y=y, Xc=Xc, alphas=np.asarray(alphas))
        for c, a in enumerate(alphas):
            m = GradientBoostingRegressor(loss="quantile", alpha=a, n_estimators=G.N_STAGES, random_state=c).fit(X, y)
            z[f"c{c}_init"] = np.float64(m.init_.constant_.ravel()[0])
            z[f"c{c}_raw"] = np.asarray([r.ravel() for r in m.staged_predict(X)])
            z[f"c{c}_pred"] = m.predict(Xc)
            for s in range(G.N_STAGES):
                t = m.estimators_[s, 0].tree_
                for k, v in (("feature", t.feature), ("threshold", t.threshold), ("left", t.children_left), ("right", t.children_right),
                             ("value", t.value[:, 0, 0]), ("n_node_samples", t.n_node_samples)):
                    z[f"c{c}_s{s}_{k}"] = np.asarray(v)
            own = G.fit_chain(X, y, a)
            z[f"c{c}_free"] = np.int32(X.shape[1] == 1 and a in EXACT and max(t["tie"] for t in own["trees"]) <= 1)
        np.savez_compressed(os.path.join(OUT, f"gbrt_{name}.npz"), **z)
        print(name, [int(z[f"c{c}_free"]) for c in range(3)])


if __name__ == "__main__":
    main()
