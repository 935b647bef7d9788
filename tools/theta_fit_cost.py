"""Cost of theta_fit="skopt" on the GPU at the workload of record (D = 32), with the card's name, power limit and max SM clock
read in the same run.  Per N: kbo_lml_grad_batch at G = 3 against three G = 1 calls (medians of synchronised host timings),
a single kbo_fit for scale (CUDA events), and the whole skopt fit (rounds, evaluations per start, wall time).  At N <= 1024 also
scikit-learn's own fit of the same data on the host, if scikit-learn is installed.  Prints one JSON line per N; ``--out PATH``
also writes the whole result as JSON.
Run:  python tools/theta_fit_cost.py [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200 import thetafit as TF
from kubeflow_b200 import workload as W
from kubeflow_b200.gp import GPEngine


def med_ms(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=None, help="write the whole result as JSON to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("theta_fit_cost needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = dict(gpu=q, host_cores=os.cpu_count(), D=32, rows=[])
    print(q, flush=True)
    eng = GPEngine(0, kernel="matern52", scratch_limit=16 << 30)
    for N in (256, 1024, 2048, 8192):
        D = 32
        X, y = W.trials(N, D)
        seed = TF.estimator_seed(0)
        thetas = [TF.theta_dict(t) for t in TF.starts(D, seed, 2)]
        reps = 10 if N <= 2048 else 5
        eng.lml_grad_batch(X, y, thetas)                                 # warm: lanes allocated, modules loaded
        b3 = med_ms(lambda: eng.lml_grad_batch(X, y, thetas), reps)
        b1 = med_ms(lambda: [eng.lml_grad_batch(X, y, [t]) for t in thetas], reps)
        fit = GPEngine(0, kernel="matern52", var_mode="auto", **W.theta_of_record(D))
        Xd, yd = torch.tensor(X, device="cuda"), torch.tensor(y, device="cuda")
        for _ in range(2):
            fit.tell(Xd, yd)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fit.tell(Xd, yd)
        e1.record()
        torch.cuda.synchronize()
        fit_ms = e0.elapsed_time(e1) / reps
        fit.close()
        walls, res = [], None
        for _ in range(3 if N <= 2048 else 2):
            t0 = time.perf_counter()
            res = TF.fit(TF.engine_batch_fn(eng, X, y), D, seed, 2)
            walls.append(time.perf_counter() - t0)
        row = dict(N=N, batch3_ms=b3, three_single_ms=b1, fit_ms=fit_ms, skopt_fit_s=float(np.median(walls)), skopt_fit_s_all=walls,
                   rounds=res.batch_calls, nfev=[s.nfev for s in res.starts], nit=[s.nit for s in res.starts],
                   status=[s.status for s in res.starts], winner=res.winner, lml=res.lml,
                   per_call=int(min(64, eng.scratch_limit // eng.lml_grad_lane_bytes(N, D, D))))
        if N <= 1024:
            try:
                from sklearn.gaussian_process import GaussianProcessRegressor
                from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel
                k = ConstantKernel(1.0, (0.01, 1000.0)) * Matern(length_scale=np.ones(D), length_scale_bounds=[(0.01, 100)] * D, nu=2.5) + WhiteKernel()
                t0 = time.perf_counter()
                g = GaussianProcessRegressor(kernel=k, alpha=1e-10, normalize_y=True, n_restarts_optimizer=2, random_state=seed).fit(X, y)
                row["sklearn_fit_s"] = time.perf_counter() - t0
                row["sklearn_lml"] = float(g.log_marginal_likelihood_value_)
            except ImportError:
                row["sklearn_fit_s"] = None
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
