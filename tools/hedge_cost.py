"""Cost of gp_hedge's sweep at cfg3 (N=8192, M=1,048,576, D=32, Matérn-5/2): EI, LCB and PI single sweeps (kbo_sweep) against
one kbo_sweep_multi for all three and one for EI + LCB (both decided at the lazy-fit stage), alternating, on the same fit and grid.  Every sweep starts from a fresh (lazy) fit, as a
suggestion does; only the sweep is timed (CUDA events).  Prints one JSON line: the card and its power limit (read in the same
run), per-variant sweep times, each kind's decision (unrefined, contenders, prefix survivors) and whether the multi sweep
returned each single sweep's suggestion."""
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from kubeflow_b200.gp import GPEngine  # noqa: E402
from oracle import gp_oracle as O  # noqa: E402

N, M, D = 8192, 1 << 20, 32
KINDS = ["ei", "lcb", "pi"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0)


def main(reps=5):
    X, y, Xc = O.synthetic(N, M, D)
    Xd = torch.tensor(Xc, device="cuda")
    e = GPEngine(0, kernel="matern52", acq="ei", var_mode="tc", **O.theta_of_record(D))

    def timed(fn, acq="ei"):
        e.acq = acq                                    # the acquisition is a fit parameter: set before the tell
        e.tell(X, y)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), r

    runs = {k: [] for k in KINDS + ["multi", "multi_ei_lcb"]}
    out = {"card": card(), "shape": [N, M, D], "reps": reps}
    for rep in range(reps + 1):                        # round 0 warms every path up and is not kept
        for k in KINDS:
            t, b = timed(lambda: e.ask(Xd), k)
            if rep:
                runs[k].append(t)
            out[f"best_{k}"] = [b.index, b.value, b.mu, b.std]
            out[f"decision_{k}"] = [e.last_unrefined(), e.last_contenders(), e.last_prefix_survivors()]
        t, bs = timed(lambda: e.ask_multi(Xd, KINDS))
        if rep:
            runs["multi"].append(t)
        out["decision_multi"] = e.last_decisions()
        t, bs2 = timed(lambda: e.ask_multi(Xd, KINDS[:2]))   # EI + LCB: both decided at the lazy-fit stage
        if rep:
            runs["multi_ei_lcb"].append(t)
        out["decision_multi_ei_lcb"] = e.last_decisions()
        out["best_multi"] = [[b.index, b.value, b.mu, b.std] for b in bs]
    out["sweep_ms"] = {k: v for k, v in runs.items()}
    out["sweep_ms_median"] = {k: float(np.median(v)) for k, v in runs.items()}
    slowest = max(out["sweep_ms_median"][k] for k in KINDS)
    out["multi_over_slowest_single"] = out["sweep_ms_median"]["multi"] / slowest
    out["multi_ei_lcb_over_slowest_single"] = out["sweep_ms_median"]["multi_ei_lcb"] / max(out["sweep_ms_median"][k] for k in KINDS[:2])
    out["multi_over_sum_of_singles"] = out["sweep_ms_median"]["multi"] / sum(out["sweep_ms_median"][k] for k in KINDS)
    out["same_suggestions"] = all(out["best_multi"][i] == out[f"best_{k}"] for i, k in enumerate(KINDS))
    out["same_suggestions_ei_lcb"] = all([b.index, b.value, b.mu, b.std] == out[f"best_{k}"] for b, k in zip(bs2, KINDS[:2]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
