"""GPU, two ranks: the SPMD server's ``tpe`` and ``multivariate-tpe`` behind a real gRPC server, with every request's
candidates sharded over the ranks.  Over ``gloo`` both ranks share cuda:0, so this runs on one GPU; over ``nccl`` each rank
has its own (skipped with fewer than two).  Without ``random_state`` both ranks' engines hold one seed, drawn on rank 0, and
the replies equal a one-process service's given that seed as ``random_state``.  A shard failure on rank 1 reaches the client
as INTERNAL, and the next request succeeds on both ranks."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ALGOS = {"tpe": {"n_startup_jobs": 3, "n_EI_candidates": 4099},
         "multivariate-tpe": {"n_startup_trials": 3, "n_ei_candidates": 4099}}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _replies(rep):
    return [[(a.name, a.value) for a in pa.assignments] for pa in rep.parameter_assignments]


def _feed(req, rep, n0, rng):
    for j, pa in enumerate(rep.parameter_assignments):
        v = {a.name: float(a.value) for a in pa.assignments}
        from tests.test_grpc_service import add_trial
        add_trial(req, f"t{n0 + j}", v, float((v["x1"] - 0.3) ** 2 + (v["x3"] - 2.0) ** 2 + 0.01 * rng.standard_normal()))
    return n0 + len(rep.parameter_assignments)


def _worker(rank, world, pg_port, backend, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(pg_port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    import grpc
    from kubeflow_b200.mvtpe import MvTpe
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.mvtpe_service import MultivariateTpeService
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.service import DispatchService
    from kubeflow_b200.suggestion.spmd import SpmdServicer
    from kubeflow_b200.suggestion.tpe_service import TpeService
    from kubeflow_b200.tpe import Tpe
    from tests.test_grpc_service import make_experiment
    defaults = {"device": dev, "shard": True}
    tpe, mv = TpeService(defaults), MultivariateTpeService(defaults)
    spmd = SpmdServicer(DispatchService([tpe, mv]))
    svc = {"tpe": tpe, "multivariate-tpe": mv}
    if rank == 1:                       # the forced failure: rank 1's shard ask raises when the flag file says so
        flag = os.path.join(os.environ["KBO_TEST_TMP"], "fail")
        for cls in (Tpe, MvTpe):
            orig = cls.ask_shard

            def ask_shard(self, *a, _orig=orig):
                if os.path.exists(flag):
                    os.unlink(flag)
                    raise RuntimeError("forced shard failure")
                return _orig(self, *a)
            cls.ask_shard = ask_shard
    res = {"rank": rank, "seeds": {}}
    if rank == 0:
        server, port = serve(spmd, port=0, host="127.0.0.1")
        ch = grpc.insecure_channel(f"127.0.0.1:{port}")
        stub = SuggestionStub(ch)
        log = {}
        for algo, settings in ALGOS.items():
            req = api.GetSuggestionsRequest(experiment=make_experiment(algo, settings, name=f"spmd-{algo}"))
            rng, n, rounds = np.random.default_rng(0), 0, []
            for rnd, k in enumerate([3, 1, 3, 3, 1, 3, 1]):
                req.current_request_number = k
                if rnd == 4:
                    open(os.path.join(os.environ["KBO_TEST_TMP"], "fail"), "w").close()
                    with pytest.raises(grpc.RpcError) as e:
                        stub.GetSuggestions(req)
                    assert e.value.code() == grpc.StatusCode.INTERNAL and "RankFailure" in e.value.details()
                    rounds.append(("failed", req.SerializeToString(), None))
                    continue
                rep = stub.GetSuggestions(req)
                assert len(rep.parameter_assignments) == k
                rounds.append((svc[algo]._exps[f"spmd-{algo}"].seed, req.SerializeToString(), _replies(rep)))
                n = _feed(req, rep, n, rng)
            log[algo] = rounds
        ch.close()
        server.stop(0)
        spmd.stop()
        # the same requests to a one-process service, random_state = the seed the sharded experiment held at each round
        single = DispatchService([TpeService({"device": dev}), MultivariateTpeService({"device": dev})])
        res["match"] = {}
        for algo, rounds in log.items():
            ok = []
            for seed, data, want in rounds:
                if want is None:
                    continue
                r = api.GetSuggestionsRequest.FromString(data)
                if not r.trials:
                    continue            # a start-up round: prior points from rank 0's generator, no engine
                s = r.experiment.spec.algorithm.algorithm_settings.add()
                s.name, s.value = "random_state", str(seed)
                r.experiment.name = f"one-{algo}-{seed}"
                ok.append(_replies(single.get_suggestions(r)) == want)
            res["match"][algo] = ok
        res["rounds"] = {a: [s for s, _, _ in r] for a, r in log.items()}
    else:
        spmd.worker_loop()
    res["seeds"] = {a: s._exps[f"spmd-{a}"].seed for a, s in svc.items()}
    res["calls"] = spmd.calls
    q.put(res)
    dist.barrier()
    dist.destroy_process_group()


def _run(backend, tmp_path):
    import torch.multiprocessing as mp
    os.environ["KBO_TEST_TMP"] = str(tmp_path)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, backend, q)) for r in range(2)]
    for p in ps:
        p.start()
    out = sorted([q.get(timeout=900) for _ in ps], key=lambda d: d["rank"])
    for p in ps:
        p.join(timeout=120)
        assert p.exitcode == 0
    r0, r1 = out
    assert r0["calls"] == r1["calls"] == 2 * 7
    assert r0["seeds"] == r1["seeds"]                      # the rebuilt experiments hold one seed on both ranks
    for algo in ALGOS:
        seeds = [s for s in r0["rounds"][algo] if s != "failed"]
        assert len(set(seeds[:4])) == 1 and len(set(seeds[4:])) == 1 and seeds[0] != seeds[4]   # rebuilt after the failure
        assert seeds[-1] == r0["seeds"][algo]
        assert r0["match"][algo] == [True] * 5, r0["match"]


def test_tpe_spmd_two_ranks_on_one_gpu_gloo(tmp_path):
    _run("gloo", tmp_path)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tpe_spmd_two_gpus_nccl(tmp_path):
    _run("nccl", tmp_path)
