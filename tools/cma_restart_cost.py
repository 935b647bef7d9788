"""One JSON line: what the CMA-ES termination test and restarts cost on the GPU.

* ask + tell per generation at (D = 128, λ = 4096) and (D = 10, λ = 10): `kbo_cma_run_synthetic` (device fitness, CUDA
  events around the whole run), median of 5 runs of 200 generations after a 20-generation warm-up.
* cma_stop_kernel's own time: torch.profiler with CUDA activities over 200 generations, mean per launch.
* kbo_cma_restart: host clock around the call (it ends in a device synchronise), same λ and λ doubled, median of 20.
* --digest: SHA-256 of X and the state after 200 generations of ask / host Rastrigin / tell without a restart, the check
  tests/test_gpu_cma_restart.py pins; runs with any libkbo that has the CmaEs ask / tell / state interface.
* --ab PARENT_TREE: cfg4 (bench.py's run_synthetic at D = 128, λ = 4096, 200 generations) generations/s of this tree and of
  PARENT_TREE, alternating, in fresh processes.
The card, its power limit and max SM clock are read in the same run."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def rastrigin(X):
    return 10.0 * X.shape[1] + (X * X - 10.0 * np.cos(2 * np.pi * X)).sum(1)


def digest(es, gens=200):
    for _ in range(gens):
        es.tell(rastrigin(es.ask().cpu().numpy()))
    X = es.ask().cpu().numpy()
    st = es.state(with_Y=True)
    h = hashlib.sha256(X.tobytes())
    for k in ("mean", "sigma", "C", "p_sigma", "pc", "B", "d", "Y"):
        h.update(np.asarray(st[k], dtype=np.float64).tobytes())
    return h.hexdigest()


DIGEST_CASES = [(128, 4096), (10, 10)]


def digests():
    from kubeflow_b200.cmaes import CmaEs
    out = {}
    for D, lam in DIGEST_CASES:
        es = CmaEs(np.full(D, 3.0), 2.0, popsize=lam, seed=7)
        out[f"{D},{lam}"] = digest(es)
        es.close()
    return out


CFG4 = ("import json, numpy as np; from kubeflow_b200.cmaes import CmaEs; es = CmaEs(np.full(128, 3.0), 2.0, popsize=4096, seed=7); "
        "es.run_synthetic('rastrigin', 20); print(json.dumps(es.run_synthetic('rastrigin', 200)))")


def ab(parent, rounds):
    res = {"this": [], "parent": []}
    for _ in range(rounds):
        for name, tree in (("parent", parent), ("this", ROOT)):
            env = dict(os.environ, PYTHONPATH=tree)
            out = subprocess.run([sys.executable, "-c", CFG4], cwd=tree, env=env, capture_output=True, text=True, check=True).stdout
            res[name].append(json.loads(out.strip().splitlines()[-1])["generations_per_s"])
    return {k: dict(generations_per_s=v, median=float(np.median(v)), spread=float(max(v) - min(v))) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--digest", action="store_true")
    ap.add_argument("--ab", metavar="PARENT_TREE")
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if a.digest:
        print(json.dumps(dict(card(), digests=digests())))
        return
    if a.ab:
        print(json.dumps(dict(card(), cfg4_ab=ab(os.path.abspath(a.ab), a.rounds))))
        return
    import torch
    from kubeflow_b200.cmaes import CmaEs
    out = card()
    for D, lam, fn in ((128, 4096, "rastrigin"), (10, 10, "sphere")):
        es = CmaEs(np.full(D, 3.0), 2.0, popsize=lam, seed=7)
        es.run_synthetic(fn, 20)
        ms = sorted(es.run_synthetic(fn, 200)["elapsed_ms"] / 200 for _ in range(5))
        prof_ms = None
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            es.run_synthetic(fn, 200)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "cma_stop_kernel" in e.key]
        if ev:
            t = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
            prof_ms = t / ev[0].count / 1e3
        rs = {}
        for name, lam2 in (("same_lambda", lam), ("lambda_doubled", min(2 * lam, 8192))):
            ts = []
            for i in range(20):
                es.restart(lam if i % 2 else lam2, np.full(D, 0.5), 0.1)   # alternate, so the growing case reallocates at most once
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                es.restart(lam2, np.full(D, 0.5), 0.1)
                ts.append((time.perf_counter() - t0) * 1e3)
            rs[name] = float(np.median(ts))
        es.close()
        out[f"d{D}_pop{lam}"] = dict(ask_tell_ms_per_generation=ms[len(ms) // 2], ask_tell_ms_min=ms[0], ask_tell_ms_max=ms[-1],
                                     stop_kernel_ms=prof_ms, restart_ms=rs)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
