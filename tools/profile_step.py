"""One warm-up + N timed suggestions at cfg3 through kbo_suggest_host — the command to run under a profiler.  Prints the library's own CUDA-event phase timings for the last step."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from kubeflow_b200.gp import GPEngine


def synthetic(N, M, D):
    """The workload of record (SURVEY.md §8(d)), restated here so that tools/ never touches oracle/."""
    X = np.random.default_rng(1234).random((N, D))
    y = np.sin(3.0 * X.sum(axis=1) / np.sqrt(D)) + 0.1 * np.random.default_rng(1235).standard_normal(N)
    Xc = np.random.default_rng(4321).random((M, D))
    return X, y, Xc


def theta_of_record(D):
    return dict(length_scale=0.3 * np.sqrt(D), amplitude=1.0, noise=1e-3, xi=0.01, kappa=1.96)


ap = argparse.ArgumentParser()
ap.add_argument("--trials", type=int, default=8192)
ap.add_argument("--candidates", type=int, default=1_048_576)
ap.add_argument("--dim", type=int, default=32)
ap.add_argument("--steps", type=int, default=1)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--var-mode", default="tc")
ap.add_argument("--k-span", type=int, default=0)
a = ap.parse_args()
X, y, _ = synthetic(a.trials, 1, a.dim)
Xc = np.random.default_rng(4321).random((a.candidates, a.dim)).astype(np.float32)
th = theta_of_record(a.dim)
eng = GPEngine(0, kernel="matern52", acq="ei", var_mode=a.var_mode, tc_k_span=a.k_span, **th)
for i in range(a.warmup + a.steps):
    best, t = eng.suggest_host(X, y, Xc)
print(json.dumps({"best": best.__dict__, "timings": t}))
