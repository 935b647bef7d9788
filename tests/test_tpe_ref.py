"""CPU: tests/_tpe_ref.py (the FP64 torch restatement the GPU tests of ``tpe`` decide against) equals the NumPy contract,
oracle/tpe_oracle.score, on random models of every parameter kind, at the edges of the range and on half-levels."""
import numpy as np
import pytest
import torch

from oracle import tpe_oracle as O
from tests import _tpe_ref as R

SPACE = [("uniform", -1.0, 3.0), ("uniform", 1e4, 1e4 + 1e-3), ("quniform", 0.0, 20.0, 1.0), ("quniform", 3.0, 48.0, 0.5),
         ("quniform", -2.5, 7.5, 0.25), ("choice", 7)]


def _history(n, seed):
    r = np.random.default_rng(seed)
    X = np.empty((n, len(SPACE)))
    for d, p in enumerate(SPACE):
        if p[0] == "uniform":
            X[:, d] = r.uniform(p[1], p[2], n)
            X[: n // 3, d] = p[1] + np.round((X[: n // 3, d] - p[1]) / (p[2] - p[1]) * 8) / 8 * (p[2] - p[1])   # ties
        elif p[0] == "quniform":
            X[:, d] = np.round(r.uniform(p[1], p[2], n) / p[3]) * p[3]
        else:
            X[:, d] = r.integers(0, p[1], n)
    return X, r.normal(size=n)


def _candidates(p, r):
    """Random points of [lo, hi), lo, the largest double below hi, and for quantized parameters every half-level x/q = j + ½
    inside the range (np.round and torch.round both round those half to even)."""
    if p[0] == "choice":
        return np.concatenate([np.arange(p[1]), r.integers(0, p[1], 50)]).astype(np.float64)
    lo, hi = p[1], p[2]
    c = [r.uniform(lo, hi, 200), [lo, np.nextafter(hi, lo)]]
    if p[0] == "quniform":
        q = p[3]
        j = np.arange(np.ceil(lo / q), np.floor(hi / q))
        half = (j + 0.5) * q
        assert (half / q == j + 0.5).all()                    # q a power of two: x/q is exact
        c += [half[(half >= lo) & (half < hi)], j * q]
    return np.concatenate(c)


@pytest.mark.parametrize("n", [0, 1, 30, 500])
def test_ref_equals_oracle(n):
    X, losses = _history(n, seed=n + 3)
    models, _ = O.build_models(SPACE, X, losses)
    r = np.random.default_rng(n)
    for d, (p, m) in enumerate(zip(SPACE, models)):
        c = _candidates(p, r)
        want = O.score(m, c)
        got = R.score(m, torch.tensor(c)).numpy()
        assert np.isfinite(want).all()
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12, err_msg=f"param {d} {p}")
        if p[0] != "choice":
            k = R.key(m, torch.tensor(c)).numpy()
            assert np.array_equal(k, c if p[0] == "uniform" else O.quantize(c, p[3]))
        if p[0] == "uniform":                                # each group's log-density, not only their difference
            for g in ("below", "above"):
                b = m[g]
                np.testing.assert_allclose(R.cont_lpdf(b, torch.tensor(c)).numpy(),
                                           O.GMM1_lpdf(c, b["w"], b["mu"], b["sigma"], p[1], p[2]), rtol=1e-12, atol=0)


def test_half_levels_round_to_even():
    m = dict(kind="quniform", q=0.5)
    x = torch.tensor([0.25, 0.75, 1.25, -0.25, 2.5 * 0.5])
    assert R.quantize(m, x).tolist() == [0.0, 1.0, 1.0, -0.0, 1.0] == O.quantize(x.numpy(), 0.5).tolist()


def test_tolerance_separates_and_pick_rule():
    """The tie rule of pick_ok: a unique best is demanded exactly, and a copy of it at a later index must not win."""
    space = [("uniform", -1.0, 3.0)]
    X, losses = np.linspace(-1, 3, 40)[:, None], (np.linspace(-1, 3, 40) - 1.0) ** 2
    m = O.build_models(space, X, losses)[0][0]
    x = torch.tensor(np.concatenate([np.linspace(-1, 3, 97), [1.0], np.linspace(-1, 3, 97)]))
    s = R.score(m, x)
    best = int(torch.argmax(s))
    assert R.pick_ok(m, x, s, best)[0]
    assert not R.pick_ok(m, x, s, best + 98)[0]                        # the later copy of the best
    assert not R.pick_ok(m, x, s, int(torch.argmin(s)))[0]
    assert float(R.tol(m, x).max()) < 1e-12
