"""GPU, one process: the shard asks of ``tpe`` and ``multivariate-tpe`` against one ``ask``.  Each simulated rank is an engine
of its own, seeded and told like the others, that asks for its ``shard_rows`` block of the candidates; the shards' (FP64
value, global index) winners are combined by the rule ``dist.global_argmax`` applies, and ``pick`` regenerates the winners.
The result must be one ask's on an identically seeded twin, bit for bit: suggestions and winning indices."""
import numpy as np
import pytest
import torch

from kubeflow_b200.dist import shard_rows
from kubeflow_b200.mvtpe import MvTpe
from kubeflow_b200.tpe import Tpe

pytestmark = pytest.mark.gpu

WORLDS = (2, 3, 8)
TPE_SPACES = {
    "uniform32": [("uniform", 0.0, 1.0)] * 32,
    "mixed": [("uniform", -3.0, 5.0), ("quniform", 0.0, 100.0, 5.0), ("choice", 4), ("uniform", 1e-3, 1.0), ("quniform", -2.0, 2.0, 0.5),
              ("choice", 2)],
}
MV_SPACES = {
    "float32": [("float", 0.0, 1.0)] * 32,
    "mixed": [("float", 0.0, 1.0)] * 28 + [("int", 0, 19, 1), ("int", 0, (1 << 18) - 1, 1), ("cat", 3), ("cat", 10)],
}
TPE_STARTUP, MV_STARTUP = 20, 10     # the services' default n_startup_jobs / n_startup_trials: the first model-based asks


def _history(space, n, seed):
    r = np.random.default_rng(seed)
    cols = []
    for p in space:
        if p[0] in ("uniform", "float"):
            cols.append(r.uniform(p[1], p[2], n))
        elif p[0] == "quniform":
            cols.append(np.round(r.uniform(p[1], p[2], n) / p[3]) * p[3])
        elif p[0] == "int":
            cols.append(p[1] + r.integers(0, int((p[2] - p[1]) // p[3]) + 1, n) * p[3])
        else:
            cols.append(r.integers(0, p[1], n).astype(float))
    return np.stack(cols, axis=1), r.standard_normal(n)


def _engine(kind, space, X, y, seed=7):
    e = Tpe(space, seed=seed) if kind == "tpe" else MvTpe(space, seed=seed)
    e.tell(X, y)
    return e


def _combine(shards):
    """dist.global_argmax's rule per row: the largest value (NaN never wins), the lowest global index among equals."""
    vals = np.stack([v.ravel() for v, _ in shards])
    idxs = np.stack([i.ravel() for _, i in shards])
    out = np.empty(vals.shape[1], np.int64)
    for j in range(vals.shape[1]):
        out[j] = -max(((v if v == v else -np.inf), -i) for v, i in zip(vals[:, j], idxs[:, j]))[1]
    return out


def _sharded(engines, k, M, world):
    shards = [e.ask_shard(k, M, *shard_rows(M, r, world)) for r, e in enumerate(engines)]
    for r, (v, i) in enumerate(shards):
        lo, hi = shard_rows(M, r, world)
        if lo == hi:
            assert np.all(v == -np.inf) and np.all(i == M)
        else:
            assert np.all((i >= lo) & (i < hi))
    win = _combine(shards)
    xs = [e.pick(k, win) for e in engines]          # every rank regenerates the winners itself
    for x in xs[1:]:
        np.testing.assert_array_equal(x, xs[0])
    return xs[0], win


def _check(kind, space, n, M, k):
    X, y = _history(space, n, 11)
    twin = _engine(kind, space, X, y)
    ref = twin.ask(k, M, return_details=True)
    for world in WORLDS:
        engines = [_engine(kind, space, X, y) for _ in range(world)]
        x, win = _sharded(engines, k, M, world)
        np.testing.assert_array_equal(win, ref["index"].ravel(), err_msg=f"world {world}")
        np.testing.assert_array_equal(x, ref["x"], err_msg=f"world {world}")
        for e in engines:
            e.close()
    twin.close()


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("M", [1, 5, 24, 4096, 1 << 20])
@pytest.mark.parametrize("n", [TPE_STARTUP, 8192])
@pytest.mark.parametrize("space", sorted(TPE_SPACES))
def test_tpe_shards_equal_one_ask(space, n, M, k):
    _check("tpe", TPE_SPACES[space], n, M, k)


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("M", [1, 5, 24, 4096, 1 << 20])
@pytest.mark.parametrize("n", [MV_STARTUP, 8192])
@pytest.mark.parametrize("space", sorted(MV_SPACES))
def test_mvtpe_shards_equal_one_ask(space, n, M, k):
    _check("mvtpe", MV_SPACES[space], n, M, k)


def test_mvtpe_shards_equal_one_ask_at_2_24():
    _check("mvtpe", MV_SPACES["float32"], 8192, 1 << 24, 1)


@pytest.mark.parametrize("M", [24, 4096, 1 << 20])
def test_tpe_two_category_ties_pick_the_first_index(M):
    """Every candidate of a two-category choice scores one of two values, so equal maxima sit in every shard: the combined
    winner must be the globally first candidate of the better category, as one ask picks it."""
    space = [("choice", 2), ("uniform", 0.0, 1.0)]
    X, y = _history(space, 200, 3)
    y = np.where(X[:, 0] == 1.0, y - 3.0, y)          # category 1 is clearly better
    twin = _engine("tpe", space, X, y)
    ref = twin.ask(4, M, return_details=True)
    cand = ref["candidates"][:, 0, :].cpu().numpy()
    for p in range(4):
        assert ref["index"][p, 0] == np.flatnonzero(cand[p] == ref["x"][p, 0])[0]
    for world in WORLDS:
        engines = [_engine("tpe", space, X, y) for _ in range(world)]
        x, win = _sharded(engines, 4, M, world)
        np.testing.assert_array_equal(win, ref["index"].ravel())
        np.testing.assert_array_equal(x, ref["x"])


@pytest.mark.parametrize("kind", ["tpe", "mvtpe"])
def test_pick_regenerates_the_ask_candidates(kind):
    """pick at any global index gives the candidate one ask drew there (quantized as the ask quantizes its winners)."""
    space = TPE_SPACES["mixed"] if kind == "tpe" else MV_SPACES["mixed"]
    X, y = _history(space, 300, 5)
    twin, eng = _engine(kind, space, X, y), _engine(kind, space, X, y)
    k, M = 3, 4096
    ref = twin.ask(k, M, return_details=True)
    cand = ref["candidates"].cpu().numpy()                  # k × D × M
    eng.ask_shard(k, M, 1000, 2000)
    rows = k * len(space) if kind == "tpe" else k
    for idx in (np.zeros(rows, np.int64), np.full(rows, M - 1), np.random.default_rng(0).integers(0, M, rows)):
        x = eng.pick(k, idx)
        ii = idx.reshape(k, -1)
        for p in range(k):
            for d, prm in enumerate(space):
                c = cand[p, d, ii[p, d] if kind == "tpe" else ii[p, 0]]
                if prm[0] == "quniform":
                    c = np.rint(c / prm[3]) * prm[3]
                assert x[p, d] == c, (p, d)
    with pytest.raises(ValueError):
        eng.pick(k, np.full(rows, M))                      # an index outside [0, n_candidates)
    with pytest.raises(ValueError):
        eng.pick(k + 1, np.zeros(rows + (len(space) if kind == "tpe" else 1), np.int64))   # not the shard ask's k


@pytest.mark.parametrize("kind", ["tpe", "mvtpe"])
def test_shard_asks_keep_the_ask_counter(kind):
    """Rounds of shard asks, with tells and an empty shard among them, stay in step with a one-GPU engine's asks."""
    space = TPE_SPACES["mixed"] if kind == "tpe" else MV_SPACES["mixed"]
    X, y = _history(space, 400, 9)
    twin = _engine(kind, space, X[:100], y[:100])
    world = 8
    engines = [_engine(kind, space, X[:100], y[:100]) for _ in range(world)]
    for rnd, (k, M) in enumerate([(2, 24), (1, 5), (3, 4096), (2, 3)]):
        if rnd == 2:
            twin.tell(X[100:], y[100:])
            for e in engines:
                e.tell(X[100:], y[100:])
        ref = twin.ask(k, M, return_details=True)
        x, win = _sharded(engines, k, M, world)
        np.testing.assert_array_equal(win, ref["index"].ravel())
        np.testing.assert_array_equal(x, ref["x"])
    engines[0].tell(X[:1], y[:1])
    with pytest.raises(ValueError):                 # a tell changes the models the winners were drawn from
        engines[0].pick(2, win)


@pytest.mark.parametrize("kind", ["tpe", "mvtpe"])
def test_shard_ask_refusals(kind):
    space = TPE_SPACES["mixed"] if kind == "tpe" else MV_SPACES["mixed"]
    X, y = _history(space, 50, 1)
    e = _engine(kind, space, X, y)
    lib = e.lib
    fn = lib.kbo_tpe_ask_shard if kind == "tpe" else lib.kbo_mvtpe_ask_shard
    rows = len(space) if kind == "tpe" else 1
    val = torch.empty(rows, dtype=torch.float64, device="cuda:0")
    idx = torch.empty(rows, dtype=torch.int64, device="cuda:0")
    cand = torch.zeros(1, len(space), 24, dtype=torch.float64, device="cuda:0")
    assert fn(e._h, e._o, 1, 24, 0, 24, cand.data_ptr(), val.data_ptr(), idx.data_ptr(), e._stream()) != 0   # cand_dev refused
    assert fn(e._h, e._o, 1, 24, 10, 5, None, val.data_ptr(), idx.data_ptr(), e._stream()) != 0               # lo > hi
    assert fn(e._h, e._o, 1, 24, 0, 25, None, val.data_ptr(), idx.data_ptr(), e._stream()) != 0               # hi > n_candidates
    with pytest.raises(ValueError):
        e.ask(1, 24, shard=True, return_details=True)
    with pytest.raises(ValueError):
        e.pick(1, np.zeros(rows, np.int64))            # no shard ask yet
    np.testing.assert_array_equal(e.ask(1, 24, shard=True), _engine(kind, space, X, y).ask(1, 24))   # one process: an ordinary ask
