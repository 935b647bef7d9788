"""One JSON line: the cost of serving ``tpe`` and ``multivariate-tpe`` with candidates sharded over the ranks of the SPMD server.

* ``per_rank``: the shard ask ONE rank runs — its M/world block of candidates — timed on one GPU, for M ∈ {2^20, 2^24} and
  world ∈ {1, 2, 4, 8}, at the shapes of ``tpe_cost.py`` / ``mvtpe_cost.py`` (n = 8192 trials, 32 floats, one point), with
  the survivors that shard decided in FP64.  The exchange and the pick are not in it.
* ``spmd_get_suggestions``: the end-to-end ``SpmdServicer.GetSuggestions`` time on rank 0 (request broadcast, every rank's
  shard ask, the all-gather over NCCL, the pick, the reply) at the default 24 candidates and at 2^20, for every rank count the
  machine's GPUs can run; the others are reported as "not measured".
The card, its power limit and max SM clock are read in the same run."""
import json
import os
import socket
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

N, D = 8192, 32
WORLDS = (1, 2, 4, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def engine(kind):
    from kubeflow_b200.mvtpe import MvTpe
    from kubeflow_b200.tpe import Tpe
    r = np.random.default_rng(0)
    e = Tpe([("uniform", 0.0, 1.0)] * D, seed=1) if kind == "tpe" else MvTpe([("float", 0.0, 1.0)] * D, seed=1)
    e.tell(r.uniform(0.0, 1.0, (N, D)), r.random(N))
    return e


def per_rank():
    from kubeflow_b200.dist import shard_rows
    out = []
    for kind in ("tpe", "multivariate-tpe"):
        e = engine("tpe" if kind == "tpe" else "mvtpe")
        for M in (1 << 20, 1 << 24):
            for world in WORLDS:
                lo, hi = shard_rows(M, 0, world)            # rank 0's block: the largest
                for _ in range(2):
                    e.ask_shard(1, M, lo, hi)                # warm-up (the first also builds the models)
                ts = []
                for _ in range(5 if M < (1 << 24) else 3):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    e.ask_shard(1, M, lo, hi)
                    ts.append((time.perf_counter() - t0) * 1e3)
                surv = e.last_survivors()
                out.append(dict(engine=kind, n=N, D=D, M=M, world=world, rank_candidates=hi - lo, per_rank_shard_ask_ms=float(np.median(ts)),
                                survivors_per_shard=int(surv.sum()), survivors_by_parameter=surv.tolist() if kind == "tpe" else None))
        e.close()
    return out


class _Ctx:
    def set_code(self, c):
        raise RuntimeError(f"GetSuggestions failed: {c}")

    def set_details(self, d):
        pass


def _spmd_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.mvtpe_service import MultivariateTpeService
    from kubeflow_b200.suggestion.service import DispatchService
    from kubeflow_b200.suggestion.spmd import SpmdServicer
    from kubeflow_b200.suggestion.tpe_service import TpeService
    d = {"device": rank, "shard": True}
    spmd = SpmdServicer(DispatchService([TpeService(d), MultivariateTpeService(d)]))
    if rank != 0:
        spmd.worker_loop()
    else:
        rows = []
        r = np.random.default_rng(0)
        X, y = r.uniform(0.0, 1.0, (N, D)), r.random(N)
        for algo, key in (("tpe", "n_EI_candidates"), ("multivariate-tpe", "n_ei_candidates")):
            for M in (24, 1 << 20):
                e = api.Experiment()
                e.name = f"cost-{algo}-{M}"
                e.spec.objective.type = api.MINIMIZE
                e.spec.objective.objective_metric_name = "loss"
                e.spec.algorithm.algorithm_name = algo
                for k, v in ((key, M), ("random_state", 3)):
                    s = e.spec.algorithm.algorithm_settings.add()
                    s.name, s.value = k, str(v)
                for j in range(D):
                    p = e.spec.parameter_specs.parameters.add()
                    p.name, p.parameter_type = f"x{j}", api.DOUBLE
                    p.feasible_space.min, p.feasible_space.max = "0.0", "1.0"
                req = api.GetSuggestionsRequest(experiment=e, current_request_number=1)
                for i in range(N):
                    t = req.trials.add()
                    t.name = f"t{i}"
                    t.spec.objective.objective_metric_name = "loss"
                    for j in range(D):
                        a = t.spec.parameter_assignments.assignments.add()
                        a.name, a.value = f"x{j}", repr(float(X[i, j]))
                    t.status.condition = api.SUCCEEDED
                    m = t.status.observation.metrics.add()
                    m.name, m.value = "loss", repr(float(y[i]))
                for _ in range(3):
                    spmd.GetSuggestions(req, _Ctx())         # warm-up: the first request tells the 8192 trials
                ts = []
                for _ in range(5):
                    t0 = time.perf_counter()
                    rep = spmd.GetSuggestions(req, _Ctx())
                    ts.append((time.perf_counter() - t0) * 1e3)
                assert len(rep.parameter_assignments) == 1
                rows.append(dict(algorithm=algo, n=N, D=D, M=M, world=world, get_suggestions_ms=float(np.median(ts))))
        spmd.stop()
        q.put(rows)
    dist.barrier()
    dist.destroy_process_group()


def spmd_rows():
    import torch.multiprocessing as mp
    out = []
    for world in WORLDS:
        if world > torch.cuda.device_count():
            out.append(dict(world=world, get_suggestions_ms="not measured", reason=f"{torch.cuda.device_count()} GPU(s) on this machine"))
            continue
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        ps = [ctx.Process(target=_spmd_worker, args=(r, world, port, q)) for r in range(world)]
        for p in ps:
            p.start()
        out += q.get(timeout=1800)
        for p in ps:
            p.join(timeout=300)
    return out


def main():
    info = card()
    print(json.dumps(dict(info, per_rank=per_rank(), spmd_get_suggestions=spmd_rows())))


if __name__ == "__main__":
    main()
