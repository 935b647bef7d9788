"""One JSON line: the RF / ET forests on the GPU — fit and sweep times (CUDA events, median after warm-up) at
(N, D, T, M) = (8192, 32, 100, 65 536), (8192, 32, 100, 2^20) and the Katib-typical (200, 8, 100, 65 536), for a single
acquisition (EI) and for the three-way gp_hedge sweep.  Beside each sweep: its node visits (M · T · mean path length, the
path lengths measured on 4096 of the candidates), the visit rate, and a stated bound — the shared-memory load issue of those
visits (one 8-byte LDS per visit and lane, a warp's 32 random-address loads taking at least 2 of the SM's 128-byte shared
memory cycles) over 132 SMs at the max SM clock.  The card, its power limit and max SM clock are read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200.forest import ForestEngine

SMS = 132


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def mean_path(eng, Xc):
    """Mean number of internal nodes a candidate passes, over trees and the given rows."""
    tot = 0
    for t in range(eng.n_trees):
        tr = eng.export(t)
        node = np.zeros(len(Xc), np.int64)
        while True:
            inner = tr["left"][node] >= 0
            if not inner.any():
                break
            r = np.flatnonzero(inner)
            tot += len(r)
            go = Xc[r, tr["feature"][node[r]]].astype(np.float64) <= tr["threshold"][node[r]]
            node[r] = np.where(go, tr["left"][node[r]], tr["right"][node[r]])
    return tot / (eng.n_trees * len(Xc))


def timed(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def measure(kind, N, D, T, M, clk):
    r = np.random.default_rng(0)
    X = r.random((N, D))
    y = np.sin(6 * X[:, 0]) + (X[:, 1:] ** 2).sum(axis=1) + 0.1 * r.standard_normal(N)
    eng = ForestEngine(kind=kind, n_trees=T, seed=1)
    fits = []
    for i in range(4):
        eng.tell(X, y + 1e-9 * i)                  # a changed history: a real refit each time
        fits.append(eng.last_timings()["fit_ms"])
    Xc = torch.rand(M, D, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    reps = 10 if M < (1 << 20) else 5
    for _ in range(2):
        eng.sweep(Xc, ["ei"])
        eng.sweep(Xc, ["ei", "lcb", "pi"])
    one = timed(lambda: eng.sweep(Xc, ["ei"]), reps)
    three = timed(lambda: eng.sweep(Xc, ["ei", "lcb", "pi"]), reps)
    depth = mean_path(eng, Xc[:4096].cpu().numpy())
    visits = M * T * (depth + 1)                   # internal nodes passed plus the leaf read
    bound_ms = visits / 32 * 2 / (SMS * clk) * 1e3
    eng.close()
    return dict(kind=kind, N=N, D=D, T=T, M=M, fit_ms=float(np.median(fits[1:])), sweep_ei_ms=one, sweep_hedge_ms=three,
                mean_path=depth, node_visits=visits, visits_per_s=visits / (one * 1e-3), lds_issue_bound_ms=bound_ms,
                share_of_bound=bound_ms / one)


def main():
    info = card()
    clk = info["max_sm_clock_mhz"] * 1e6
    rows = []
    for kind in ("RF", "ET"):
        for N, D, T, M in ((8192, 32, 100, 65536), (8192, 32, 100, 1 << 20), (200, 8, 100, 65536)):
            t0 = time.perf_counter()
            rows.append(measure(kind, N, D, T, M, clk))
            rows[-1]["wall_s"] = time.perf_counter() - t0
    print(json.dumps(dict(info, shapes=rows)))


if __name__ == "__main__":
    main()
