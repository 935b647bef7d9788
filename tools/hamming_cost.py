"""Cost of kernel="hamming" on the GPU, beside Matérn on the same one-hot columns, with the card's name, power limit and max SM
clock read in the same run.  D = 32 categorical dimensions with 1, 2, 3 and 7 categories (96 one-hot columns), the history
of tests/test_gpu_hamming.py.  Per N ∈ {256, 2048, 8192}:
  fit_ms        one kbo_fit at the default θ (CUDA events, median of reps)
  theta_fit_s   the whole theta_fit="skopt" fit (three starts in lockstep; wall time, one run, after one untimed batch and
                SciPy's import), and round_ms = theta_fit_s / rounds
  ask_ms[M]     one suggestion (array-free sweep, EI) over M ∈ {65 536, 2²⁰} float32 candidates already on the device (CUDA events)
for the Hamming kernel at its default weights (l_j = 1, in the tensor-core range), for Matérn-5/2 at the default length scale
0.3·√96, and for the Hamming kernel on the FP64 route (var_mode "f64", what "auto" takes outside the tensor-core range).
Prints one JSON line per N; ``--out PATH`` also writes the whole result as JSON.
Run:  python tools/hamming_cost.py [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200 import hamming as HM
from kubeflow_b200 import thetafit as TF
from kubeflow_b200.gp import GPEngine
from kubeflow_b200.space import Categorical, Space

CATS = [1, 2, 3, 7] * 8


def events_ms(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=None, help="write the whole result as JSON to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hamming_cost needs a CUDA device")
    import scipy.optimize  # noqa: F401  (imported inside the first fit otherwise, and timed with it)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(q, flush=True)
    sp = Space([Categorical(list(range(c)), name=f"c{j}") for j, c in enumerate(CATS)])
    hm = HM.HammingMap(sp)
    Dt = sp.transformed_n_dims
    out = dict(gpu=q, D=len(CATS), columns=Dt, rows=[])
    r = np.random.default_rng(0)
    grids = {M: torch.as_tensor(sp.rvs_transformed(M, np.random.default_rng(M), np.float32), device="cuda") for M in (65536, 1 << 20)}
    seed = TF.estimator_seed(0)
    models = {"hamming": dict(kernel="rbf", length_scale=hm.length_scale(1.0), var_mode=hm.var_mode(1.0, "auto")),
              "matern_one_hot": dict(kernel="matern52", length_scale=0.3 * np.sqrt(Dt), var_mode="auto"),
              "hamming_f64": dict(kernel="rbf", length_scale=hm.length_scale(1.0), var_mode="f64")}
    for N in (256, 2048, 8192):
        X = sp.rvs_transformed(N, r, np.float64)
        codes = np.stack([X[:, hm.col_dim == j].argmax(1) if CATS[j] > 2 else X[:, hm.col_dim == j][:, 0] for j in range(len(CATS))], 1)
        y = np.sin(codes[:, 1:9] @ np.linspace(0.2, 1.0, 8)) + 0.1 * r.standard_normal(N)
        Xd, yd = torch.tensor(X, device="cuda"), torch.tensor(y, device="cuda")
        row = dict(N=N)
        reps = 5 if N <= 2048 else 3
        for name, kw in models.items():
            e = GPEngine(0, acq="ei", noise=1e-3, scratch_limit=16 << 30, **kw)
            res = dict(fit_ms=events_ms(lambda: e.tell(Xd, yd), reps))
            for M, G in grids.items():
                res[f"ask_ms_{M}"] = events_ms(lambda: e.ask(G), reps if name != "hamming_f64" else 2)
            if name != "hamming_f64":
                bfn = TF.engine_batch_fn(e, X, y, hamming=hm if name == "hamming" else None)
                bfn([np.zeros(2 + (len(CATS) if name == "hamming" else Dt))] * 3)      # warm: lanes allocated, modules loaded
                t0 = time.perf_counter()
                fr = TF.fit(TF.engine_batch_fn(e, X, y, hamming=hm if name == "hamming" else None), len(CATS) if name == "hamming" else Dt,
                            seed, 2, ls_bounds=HM.LS_BOUNDS if name == "hamming" else TF.LS_BOUNDS)
                res.update(theta_fit_s=time.perf_counter() - t0, rounds=fr.batch_calls,
                           round_ms=(time.perf_counter() - t0) * 1e3 / fr.batch_calls, nfev=[s.nfev for s in fr.starts], lml=fr.lml)
            e.close()
            row[name] = res
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
