"""Histories and candidate grids at the shapes the engine serves, shared by test_gpu_grid_scale.py and test_gpu_rank_rows.py.

Every case is at the θ of record (oracle.theta_of_record) unless its entry says otherwise.  ``grid`` says how the candidates
reach the engine: "cuda32" a float32 CUDA tensor, "host32" / "host64" a NumPy array.
"""
import numpy as np
import torch

from kubeflow_b200 import workload as W
from oracle import gp_oracle as O

M3 = 1_048_576

CASES = {
    "cfg3": dict(kind="matern52", N=8192, D=32, M=M3, grid="cuda32"),
    "cfg3-raw-y": dict(kind="matern52", N=8192, D=32, M=1_048_539, grid="host64", y=(2e4, 5.0)),
    "cfg3-ard": dict(kind="matern52", N=8192, D=32, M=M3, grid="host32", ard=(0.5, 2.0)),
    "n4097-rbf": dict(kind="rbf", N=4097, D=32, M=1_000_003, grid="cuda32"),
    "cfg2": dict(kind="rbf", N=1024, D=8, M=65_536, grid="cuda32"),
    "near-trials-1e-3": dict(kind="matern52", N=8192, D=32, M=M3, grid="host64", noise=1e-3, near=4096),
    "near-trials-1e-6": dict(kind="matern52", N=8192, D=32, M=M3, grid="host64", noise=1e-6, near=4096),
    # the widest tensor-core K* (four 32-feature slabs)
    "d128": dict(kind="matern52", N=8192, D=128, M=262_144, grid="cuda32"),
    # the amplitude at which DESIGN.md §1 records the largest tensor-core array errors
    "amp-1e3": dict(kind="matern52", N=8192, D=32, M=M3, grid="cuda32", amplitude=1e3),
    # long length scales with little noise: the conditioning `auto` cannot detect, and the largest tensor-core array errors
    # DESIGN.md §1 records
    "ls5-noise-1e-6": dict(kind="matern52", N=8192, D=32, M=M3, grid="cuda32", ls_mult=5.0, noise=1e-6),
    # a late-stage experiment on few hyperparameters: ¾ of the trials in a ball of radius 0.03 around x₀,
    # y = 10‖x − x₀‖² + 0.1·noise; 16,384 of the candidates within 0.06 of x₀
    "converged-d4": dict(kind="matern52", N=4096, D=4, M=M3, grid="cuda32", converged=(0.03, 16_384)),
}


def _ball(r, n, D, radius):
    """n points uniform in the D-ball of the given radius around 0."""
    u = r.standard_normal((n, D))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return u * (radius * r.random((n, 1)) ** (1.0 / D))


def case_data(name):
    """dict(name, kind, X, y, Xc, M, theta, near (rows replaced by trial copies / near-copies, or None), tc)."""
    c = CASES[name]
    N, D, M = c["N"], c["D"], c["M"]
    X, y, _ = O.synthetic(N, 1, D)
    if "y" in c:
        y = c["y"][0] + c["y"][1] * y
    th = O.theta_of_record(D)
    if "ard" in c:
        th["length_scale"] = th["length_scale"] * np.linspace(*c["ard"], D)
    if "ls_mult" in c:
        th["length_scale"] = th["length_scale"] * c["ls_mult"]
    for k in ("noise", "amplitude"):
        if k in c:
            th[k] = c[k]
    Xc = W.candidates(M, D, dtype=np.float64 if c["grid"] == "host64" else np.float32)
    near = None
    if "converged" in c:
        radius, n_near = c["converged"]
        r = np.random.default_rng(23)
        x0 = 0.2 + 0.6 * r.random(D)
        k = 3 * N // 4
        X[:k] = x0 + _ball(r, k, D, radius)
        y = 10.0 * ((X - x0) ** 2).sum(1) + 0.1 * r.standard_normal(N)
        rows = r.choice(M, n_near, replace=False)
        Xc[rows] = (x0 + _ball(r, n_near, D, 2 * radius)).astype(Xc.dtype)
    if "near" in c:
        r = np.random.default_rng(17)
        n = c["near"]
        near = r.choice(M, 2 * n, replace=False)
        Xc[near[:n]] = X[r.choice(N, n, replace=False)]
        Xc[near[n:]] = X[r.choice(N, n, replace=False)] + 1e-7 * (2 * r.random((n, D)) - 1)
    if c["grid"] == "cuda32":
        Xc = torch.tensor(Xc, device="cuda")
    return dict(name=name, kind=c["kind"], X=X, y=y, Xc=Xc, M=M, theta=th, near=near, tc=name != "cfg2")
