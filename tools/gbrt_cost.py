"""One JSON line: skopt's GBRT surrogate on the GPU — fit and sweep times (CUDA events, median after warm-up) at (N, D) = (200, 8)
and (8192, 32), each swept at M = 65 536 and 2^20 candidates, for EI alone and for the three-way gp_hedge sweep.  Beside each
sweep: the bytes of its one read of the candidates (M·D·4) and that read's time at the 3.35 TB/s HBM3 data-sheet bandwidth, the
bound the sweep is reported against.  The card, its power limit and max SM clock are read in the same run."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200.gbrt import GbrtEngine

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def timed(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def measure(N, D):
    r = np.random.default_rng(0)
    X = r.random((N, D))
    y = np.sin(6 * X[:, 0]) + (X[:, 1:] ** 2).sum(axis=1) + 0.1 * r.standard_normal(N)
    eng = GbrtEngine()
    eng.tell(X, y)
    fits = []
    for i in range(5):
        eng._hist = None                      # force a refit of the same history
        eng.tell(X, y)
        fits.append(eng.last_timings()["fit_ms"])
    out = dict(N=N, D=D, fit_ms=float(np.median(fits[1:])), sweeps=[])
    dev = torch.device("cuda", 0)
    for M in (65536, 1 << 20):
        Xc = torch.rand((M, D), device=dev, dtype=torch.float32)
        row = dict(M=M)
        for name, acqs in (("ei", ["ei"]), ("hedge", ["ei", "lcb", "pi"])):
            for _ in range(3):
                eng.sweep(Xc, acqs)
            row[f"{name}_ms"] = timed(lambda: eng.sweep(Xc, acqs), 20)
        row["read_bytes"] = M * D * 4
        row["read_bound_ms"] = M * D * 4 / HBM * 1e3
        out["sweeps"].append(row)
    eng.close()
    return out


def main():
    res = dict(card=card(), cases=[measure(200, 8), measure(8192, 32)])
    print(json.dumps(res))
    od = os.environ.get("GBRT_COST_OUT")
    if od:
        with open(od, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
