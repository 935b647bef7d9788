"""One JSON line: the TPE ask on the GPU at n = 8192 trials, D = 32 continuous parameters, M ∈ {24, 4096, 2^20} candidates —
per-phase CUDA-event times after warm-up, survivor counts, the score kernel's MUFU and FP32-issue bounds computed from shapes,
and the FP64 NumPy oracle's ask time on this host's cores (at M = 2^20 timed on a subsample and extrapolated linearly in M,
labelled so).  The card, its power limit and max SM clock are read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200.tpe import Tpe
from oracle import tpe_oracle as O

N, D = 8192, 32
SMS, EX2_PER_CLK, FP32_PER_CLK = 132, 16, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def main():
    info = card()
    r = np.random.default_rng(0)
    space = [("uniform", 0.0, 1.0)] * D
    X, y = r.random((N, D)), r.random(N)
    t = Tpe(space, seed=1)
    t.tell(X, y)
    models, nb = O.build_models(space, X, y)
    out = dict(info, n=N, D=D, n_below=nb, shapes=[])
    clk = info["max_sm_clock_mhz"] * 1e6
    for M in (24, 4096, 1 << 20):
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
        exps = D * M * (N + 2)                           # one ex2 per component per candidate (below: n_below + 1, above: N - n_below + 1)
        mufu_ms = exps / (SMS * EX2_PER_CLK * clk) * 1e3
        fp32_ms = 11 * exps / (SMS * FP32_PER_CLK * clk) * 1e3   # 11 FP32-pipe instructions per term (two passes per staged chunk)
        sub = min(M, 4096)
        cands = [O.draw(m, sub, r) for m in models]
        c0 = time.perf_counter()
        O.choose(models, cands)
        cpu_ms = (time.perf_counter() - c0) * 1e3 * (M / sub)
        out["shapes"].append(dict(M=M, phases_ms=med, survivors=t.last_survivors().tolist(), mufu_bound_ms=mufu_ms, fp32_issue_bound_ms=fp32_ms,
                                  score_share_of_mufu_bound=mufu_ms / med["score_fp32_ms"] if med["score_fp32_ms"] else None,
                                  cpu_oracle_ms=cpu_ms, cpu_oracle_extrapolated=M > sub, cpu_threads=os.cpu_count()))
    t.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
