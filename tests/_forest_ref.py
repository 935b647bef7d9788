"""Shared by the forest tests: tree comparison by a walk from the root (sklearn numbers nodes depth-first, the device and the
restatement breadth-first) and the golden cases."""
from __future__ import annotations

import glob
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_cases():
    return sorted(glob.glob(os.path.join(GOLDEN, "forest_*.npz")))


def golden_trees(z):
    keys = ("feature", "threshold", "left", "right", "value", "impurity", "n_node_samples", "weighted_n_node_samples")
    return [{k: z[f"t{t}_{k}"] for k in keys} for t in range(int(z["n_trees"]))]


def assert_same_tree(a, b, rtol=1e-12, where=""):
    """Same structure, features, bit-equal thresholds, equal distinct / weighted counts; value and impurity to rtol (0: bit-equal).
    The impurity Σ(w·y)·y / Σw − value² cancels where the spread of y is small against its mean, so its sums taken in another
    order move it by rtol relative to the terms that cancel: it is compared against max(|impurity|, value²)."""
    stack = [(0, 0)]
    seen = 0
    while stack:
        i, j = stack.pop()
        seen += 1
        ctx = f"{where} node a{i}/b{j}"
        la, lb = int(a["left"][i]), int(b["left"][j])
        assert (la < 0) == (lb < 0), f"{ctx}: leaf in one tree only"
        assert int(a["n_node_samples"][i]) == int(b["n_node_samples"][j]), ctx
        assert float(a["weighted_n_node_samples"][i]) == float(b["weighted_n_node_samples"][j]), ctx
        for k in ("value", "impurity"):
            va, vb = float(a[k][i]), float(b[k][j])
            if rtol == 0:
                assert va == vb, f"{ctx}: {k} {va!r} != {vb!r}"
            else:
                scale = max(abs(va), abs(vb), float(a["value"][i]) ** 2 if k == "impurity" else 0.0, 1e-300)
                assert abs(va - vb) <= rtol * scale, f"{ctx}: {k} {va!r} vs {vb!r}"
        if la >= 0:
            assert int(a["feature"][i]) == int(b["feature"][j]), f"{ctx}: feature"
            assert float(a["threshold"][i]) == float(b["threshold"][j]), f"{ctx}: threshold {a['threshold'][i]!r} vs {b['threshold'][j]!r}"
            stack += [(int(a["right"][i]), int(b["right"][j])), (la, lb)]
    assert seen == len(a["left"]) == len(b["left"]), f"{where}: node counts {len(a['left'])} vs {len(b['left'])}"


def dyadic_case(rng, N, D, *, grid=False):
    """X in [0, 1) (float32) and y on a grid of 2^-12 in [-4, 4]: every weighted sum and square is exact in FP64, so split
    proxies do not depend on the order sums are taken in and equal partitions tie exactly on device and restatement."""
    X = rng.random((N, D)).astype(np.float32)
    if grid:
        X[:, 0] = rng.integers(0, 9, N) / 8.0            # integer parameter
        X[:, 1] = rng.integers(0, 2, N)                  # one-hot column
    y = np.sin(4.0 * X[:, 0]) + X[:, -1] ** 2 + 0.3 * rng.standard_normal(N)
    y = np.clip(np.round(y * 4096.0), -16384, 16384) / 4096.0
    return X, y
