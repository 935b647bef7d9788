"""CPU, world_size 2 over gloo: the host side of the sharded ``tpe`` / ``multivariate-tpe`` ask (``dist.sharded_ask``) and of
the services that use it under SPMD.  The engines are test-only stand-ins, so what is tested is the exchange: the combine
rule with empty shards, -inf and first-index ties across ranks; a raising rank making every rank raise ``RankFailure``;
seeds agreeing across ranks; a failed experiment closed on every rank.  And ``shard`` is never an Experiment setting."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from kubeflow_b200.suggestion.internal import AlgorithmSettingsError


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(target, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=target, args=(r, port, q) + args) for r in range(2)]
    for p in ps:
        p.start()
    out = sorted([q.get(timeout=300) for _ in ps], key=lambda d: d["rank"])
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


def _init(rank, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2")
    dist.init_process_group("gloo", rank=rank, world_size=2)


# rows of (rank 0's (value, index), rank 1's (value, index)) with n_candidates = 10 (rank 0 owns [0, 5), rank 1 [5, 10))
# and the winning index
CASES = [
    (((1.0, 2), (2.0, 7)), 7),                           # the larger value
    (((3.0, 4), (3.0, 5)), 4),                           # equal values across ranks: the first index
    (((-np.inf, 0), (-np.inf, 9)), 0),                   # every candidate -inf: still the first index
    (((-np.inf, 3), (-np.inf, 10)), 3),                  # an empty shard's (-inf, n_candidates) never wins, even against -inf
    (((np.nan, 1), (0.5, 6)), 6),                        # NaN never wins
    (((-5.0, 0), (-np.inf, 10)), 0),
]


def _combine_worker(rank, port, q):
    _init(rank, port)
    from kubeflow_b200.dist import RankFailure, sharded_ask, shard_rows
    seen = {}

    def shard(lo, hi):
        seen["rows"] = (lo, hi)
        return np.array([c[0][rank][0] for c in CASES]), np.array([c[0][rank][1] for c in CASES], np.int64)

    res = dict(rank=rank, win=sharded_ask(shard, lambda idx: list(idx), 10, len(CASES), torch.device("cpu")))
    res["rows"] = seen["rows"]
    assert shard_rows(10, rank, 2) == seen["rows"]

    def fail(lo, hi):
        if rank == 1:
            raise RuntimeError("forced shard failure")
        return shard(lo, hi)

    try:
        sharded_ask(fail, lambda idx: pytest.fail("picked after a failure"), 10, len(CASES), torch.device("cpu"))
        res["raised"] = None
    except RankFailure as e:
        res["raised"] = str(e)
    q.put(res)
    dist.destroy_process_group()


def test_sharded_ask_combine_rule_and_rank_failure():
    r0, r1 = _run(_combine_worker)
    want = [c[1] for c in CASES]
    assert r0["win"] == r1["win"] == want
    assert r0["rows"] == (0, 5) and r1["rows"] == (5, 10)
    assert "rank(s) [1]" in r0["raised"] and "forced shard failure" in r1["raised"]


class _FakeTpe:
    """Stands in for kubeflow_b200.tpe.Tpe: candidate m of a point scores a hash of (seed, ask, point, m) and sits at a value
    computed from m, so a sharded ask's winner is known; ``fail`` makes the next shard ask raise."""
    made, fail = [], False

    def __init__(self, space, seed, **_):
        self.space, self.seed, self.asks, self.n, self.closed = space, seed, 0, 0, False
        _FakeTpe.made.append(self)

    def tell(self, X, y):
        self.n += len(X)

    def _score(self, ask, k, ms):
        h = (np.uint64(self.seed % (1 << 40)) * np.uint64(2654435761) + np.uint64(ask * 1000003)
             + np.arange(k, dtype=np.uint64)[:, None] * np.uint64(7919) + np.asarray(ms, np.uint64)[None, :] * np.uint64(104729))
        return ((h * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(40)).astype(np.float64)

    def _x(self, k, idx, M):
        return [[lo + (hi - lo) * (i + 0.5) / M for (_, lo, hi) in self.space] for i in np.asarray(idx).reshape(k)]

    def ask(self, k, M, shard=False):
        from kubeflow_b200.dist import sharded_ask
        ask = self.asks
        self.asks += 1
        if not shard or dist.get_world_size() == 1:
            s = self._score(ask, k, range(M))
            return np.asarray(self._x(k, s.argmax(1), M))

        def shard_fn(lo, hi):
            if _FakeTpe.fail:
                _FakeTpe.fail = False
                raise RuntimeError("forced shard failure")
            if lo == hi:
                return np.full(k, -np.inf), np.full(k, M, np.int64)
            s = self._score(ask, k, range(lo, hi))
            return s.max(1), lo + s.argmax(1)
        return np.asarray(sharded_ask(shard_fn, lambda idx: self._x(k, idx, M), M, k, torch.device("cpu")))

    def close(self):
        self.closed = True


def _service_worker(rank, port, q):
    _init(rank, port)
    import kubeflow_b200.tpe
    kubeflow_b200.tpe.Tpe = _FakeTpe
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.tpe_service import TpeService
    from tests.test_grpc_service import add_trial, make_experiment
    svc = TpeService({"shard": True})
    single = TpeService()
    exp = make_experiment("tpe", {"n_startup_jobs": 2, "n_EI_candidates": 7}, name="shard")
    req = api.GetSuggestionsRequest(experiment=exp, current_request_number=3)
    for i in range(3):
        add_trial(req, f"t{i}", {"x0": 0.05, "x1": 0.1 * i, "x2": 12.0, "x3": float(i)}, float(i))
    res = dict(rank=rank, replies=[])
    for rnd in range(4):
        if rnd == 2 and rank == 1:
            _FakeTpe.fail = True
        try:
            rep = svc.get_suggestions(req)
            res["replies"].append([[a.value for a in pa.assignments] for pa in rep.parameter_assignments])
        except Exception as e:  # noqa: BLE001
            res["replies"].append(type(e).__name__)
    res["seeds"] = [e.seed for e in _FakeTpe.made]
    res["closed"] = [e.closed for e in _FakeTpe.made]
    # the same requests to a one-process service with the shared seed as random_state: the same replies
    exp1 = make_experiment("tpe", {"n_startup_jobs": 2, "n_EI_candidates": 7, "random_state": res["seeds"][0]}, name="one")
    req1 = api.GetSuggestionsRequest(experiment=exp1, current_request_number=3)
    req1.trials.extend(req.trials)
    _FakeTpe.made = []
    res["single"] = [[[a.value for a in pa.assignments] for pa in single.get_suggestions(req1).parameter_assignments] for _ in range(2)]
    q.put(res)
    dist.destroy_process_group()


def test_tpe_service_sharded_seeds_and_failure():
    r0, r1 = _run(_service_worker)
    assert r0["seeds"] == r1["seeds"] and len(r0["seeds"]) == 2       # no random_state: one seed, drawn on rank 0, everywhere
    assert r0["replies"] == r1["replies"]
    assert r0["replies"][2] == r1["replies"][2] == "RankFailure"      # rank 1's failure fails the request on both ranks …
    assert r0["closed"] == r1["closed"] == [True, False]              # … closes the experiment on both, and the next request
    assert isinstance(r0["replies"][3], list) and len(r0["replies"][3]) == 3   # rebuilds it alike everywhere
    assert r0["replies"][:2] == r0["single"]                          # sharded replies = one process's, same seed
    assert r0["replies"][0] != r0["replies"][1]


@pytest.mark.parametrize("algorithm", ["tpe", "multivariate-tpe"])
def test_shard_is_not_an_experiment_setting(algorithm):
    from kubeflow_b200.suggestion.mvtpe_service import MultivariateTpeService
    from kubeflow_b200.suggestion.tpe_service import TpeService
    from tests.test_grpc_service import make_experiment
    svc = TpeService({"shard": True}) if algorithm == "tpe" else MultivariateTpeService({"shard": True})
    with pytest.raises(AlgorithmSettingsError, match="unknown setting shard"):
        svc.validate(make_experiment(algorithm, {"shard": "true"}))
