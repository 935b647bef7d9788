"""CPU: oracle/forest_oracle.py — the FP64 restatement of the RF / ET surrogates — against trees the real scikit-learn 1.9.0
fitted (tests/golden/forest_*.npz, written by oracle/make_golden_forest.py), and its Philox draws and ET rules on their own."""
import numpy as np
import pytest

from oracle import forest_oracle as F
from tests._forest_ref import assert_same_tree, dyadic_case, golden_cases, golden_trees


@pytest.mark.parametrize("path", golden_cases(), ids=lambda p: p.rsplit("/", 1)[-1])
def test_restatement_reproduces_every_golden_tree(path):
    z = np.load(path)
    ref = golden_trees(z)
    mine = [F.build_tree(z["X"], z["y"], z["counts"][t], min_samples_leaf=3, kind="RF") for t in range(len(ref))]
    for t, (a, b) in enumerate(zip(mine, ref)):
        assert_same_tree(a, b, rtol=1e-12, where=f"tree {t}")
    mu, sd = F.predict(mine, z["Xc"])
    np.testing.assert_allclose(mu, z["mu"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(sd, z["sigma"], rtol=1e-12, atol=1e-12)


def test_golden_counts_are_the_philox_bootstrap():
    for path in golden_cases():
        z = np.load(path)
        N = len(z["y"])
        for t, seed in enumerate(z["seeds"]):
            assert np.array_equal(z["counts"][t], F.bootstrap_counts(N, t + 1, int(seed))[t])


def test_bootstrap_counts_draw_n_samples_uniformly():
    c = F.bootstrap_counts(1000, 50, 123)
    assert c.shape == (50, 1000) and (c.sum(axis=1) == 1000).all()
    from scipy import stats
    # per tree, the count of a sample is Binomial(N, 1/N); pooled over 50 trees the share of unseen samples is near e^-1
    assert abs((c == 0).mean() - np.exp(-1)) < 0.01
    assert stats.chisquare(c.sum(axis=0).reshape(50, 20).sum(axis=1)).pvalue > 1e-3
    assert not np.array_equal(c[0], c[1]) and not np.array_equal(F.bootstrap_counts(1000, 1, 124)[0], c[0])


def test_et_uniform_and_threshold_rule():
    from scipy import stats
    u = F.et_uniform(5, 3, np.arange(20000), 7)
    assert (u >= 0).all() and (u < 1).all()
    assert stats.kstest(u, "uniform").pvalue > 1e-3
    assert F.et_threshold(1.0 - 2.0 ** -53, np.float32(0.25), np.float32(0.5)) == 0.25   # equals max: min
    mn, mx = np.float32(0.1), np.float32(0.7)
    th = F.et_threshold(u, mn, mx)
    assert (th >= np.float64(mn)).all() and (th < np.float64(mx)).all()


def test_et_tree_rules_hold():
    rng = np.random.default_rng(3)
    X, y = dyadic_case(rng, 400, 5, grid=True)
    tree = F.build_forest(X, y, kind="ET", n_trees=1, seed=9)[0]
    leaf = F.apply(tree, X)
    inner = np.flatnonzero(tree["left"] >= 0)
    assert len(inner) > 10
    assert (tree["n_node_samples"][tree["left"] < 0] >= 3).all()
    assert np.array_equal(np.bincount(leaf, minlength=len(tree["left"]))[tree["left"] < 0], tree["n_node_samples"][tree["left"] < 0])
    assert (tree["weighted_n_node_samples"] == tree["n_node_samples"]).all()


def test_predict_is_skopt_return_std():
    rng = np.random.default_rng(1)
    X, y = dyadic_case(rng, 120, 3)
    trees = F.build_forest(X, y, kind="RF", n_trees=7, seed=2)
    Xc = rng.random((50, 3)).astype(np.float32)
    mu, sd = F.predict(trees, Xc)
    V = np.array([t["value"][F.apply(t, Xc)] for t in trees])
    I = np.maximum(np.array([t["impurity"][F.apply(t, Xc)] for t in trees]), 0.0)
    np.testing.assert_allclose(mu, V.mean(axis=0), rtol=1e-14)
    np.testing.assert_allclose(sd, np.sqrt(np.maximum((I + V ** 2).mean(axis=0) - V.mean(axis=0) ** 2, 0)), rtol=1e-9, atol=1e-12)


def test_single_sample_and_constant_y_give_single_leaf_trees():
    X = np.array([[0.5, 0.5]], np.float32)
    t = F.build_tree(X, np.array([2.0]), np.array([1]))
    assert len(t["left"]) == 1 and t["value"][0] == 2.0
    rng = np.random.default_rng(0)
    X = rng.random((50, 2)).astype(np.float32)
    t = F.build_tree(X, np.full(50, 0.75), None)
    assert len(t["left"]) == 1 and t["impurity"][0] == 0.0


def test_acquisitions_are_zero_where_sigma_is_zero():
    mu, sd = np.array([0.0, 1.0, -1.0]), np.array([0.0, 0.5, 0.0])
    assert F.acquisition("ei", mu, sd, 0.0)[0] == 0.0 and F.acquisition("pi", mu, sd, 0.0)[2] == 0.0
    assert F.acquisition("lcb", mu, sd, 0.0, kappa=2.0)[1] == -(1.0 - 1.0)
    from scipy import stats
    z = (0.0 - 0.01 - 1.0) / 0.5
    np.testing.assert_allclose(F.acquisition("ei", mu, sd, 0.0)[1], (-1.01) * stats.norm.cdf(z) + 0.5 * stats.norm.pdf(z), rtol=1e-14)
