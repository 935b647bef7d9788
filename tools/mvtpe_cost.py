"""One JSON line: the multivariate TPE ask on the GPU — per-phase CUDA-event times after warm-up and survivor counts — for one
point at n = 8192 trials over D = 32 float parameters with M ∈ {24, 4096, 2^20} candidates, and over a mixed space (28
floats, integers of 20 and 2^18 levels, two categoricals) at M = 4096.  Beside each: the score kernel's bounds computed from
shapes, 2·M·(n + 1)·D_float FP32-pipe instructions over 132 SMs × 128 lanes × clock and M·(n + 1) exponentials over 132 SMs ×
16 per clock.  The card, its power limit and max SM clock are read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200.mvtpe import MvTpe

N = 8192
SMS, EX2_PER_CLK, FP32_PER_CLK = 132, 16, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def history(space, r):
    cols = []
    for p in space:
        if p[0] == "float":
            cols.append(r.uniform(p[1], p[2], N))
        elif p[0] == "int":
            cols.append(p[1] + r.integers(0, int((p[2] - p[1]) // p[3]) + 1, N) * p[3])
        else:
            cols.append(r.integers(0, p[1], N).astype(float))
    return np.stack(cols, axis=1), r.random(N)


def measure(name, space, Ms, clk):
    r = np.random.default_rng(0)
    X, y = history(space, r)
    t = MvTpe(space, seed=1)
    t.tell(X, y)
    df = sum(p[0] == "float" for p in space)
    out = []
    for M in Ms:
        for _ in range(3):
            t.ask(1, M)                                  # warm-up (the first ask also builds the models)
        reps = 5 if M < (1 << 20) else 3
        ph = []
        for _ in range(reps):
            torch.cuda.synchronize()
            w0 = time.perf_counter()
            t.ask(1, M)
            ph.append(dict(t.last_timings(), wall_ms=(time.perf_counter() - w0) * 1e3))
        med = {k: float(np.median([p[k] for p in ph])) for k in ph[0]}
        pairs = M * (N + 1)
        fp32_ms = 2 * pairs * df / (SMS * FP32_PER_CLK * clk) * 1e3
        mufu_ms = pairs / (SMS * EX2_PER_CLK * clk) * 1e3
        out.append(dict(workload=name, n=N, D=len(space), D_float=df, M=M, phases_ms=med, survivors=t.last_survivors().tolist(),
                        fp32_issue_bound_ms=fp32_ms, mufu_bound_ms=mufu_ms,
                        score_share_of_fp32_bound=fp32_ms / med["score_fp32_ms"] if med["score_fp32_ms"] else None))
    t.close()
    return out


def main():
    info = card()
    clk = info["max_sm_clock_mhz"] * 1e6
    rows = measure("float32", [("float", 0.0, 1.0)] * 32, (24, 4096, 1 << 20), clk)
    mixed = [("float", 0.0, 1.0)] * 28 + [("int", 0, 19, 1), ("int", 0, (1 << 18) - 1, 1), ("cat", 3), ("cat", 10)]
    rows += measure("mixed", mixed, (4096,), clk)
    print(json.dumps(dict(info, shapes=rows)))


if __name__ == "__main__":
    main()
