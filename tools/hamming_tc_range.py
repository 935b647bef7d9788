"""Where the tensor-core sweep holds for Hamming weights: the evidence behind ``kubeflow_b200.hamming.TC_RANGE``.

At the history and grid of tests/test_gpu_hamming.py (D = 32 categorical dimensions with 1, 2, 3 and 7 categories, 24 of which
can differ; N = 2048, M = 65 536), equal weights l_j = S / 24 for a range of S, and each of EI and LCB: the engine sweeps in
var_mode "auto" whatever TC_RANGE says (so the tensor cores run wherever auto's size rule allows), and its pick is compared
with the FP64 oracle's argmax over every candidate.  ``held`` is true when the pick is the oracle's first argmax or within
1e-9 (relative) of its value; ``shortfall`` is (max − value at the pick) / max(1, |max|).  Prints one JSON line per (S, acq)
with the card's name, power limit and max SM clock read in the same run.
Run:  python tools/hamming_tc_range.py [--s 0.05 0.1 ...]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from tests import test_gpu_hamming as T
from oracle import hamming_oracle as H
from kubeflow_b200.gp import GPEngine


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--s", type=float, nargs="*", default=[0.05, 0.1, 0.255, 1.0, 4.0, 16.0, 31.4, 64.0, 125.0])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hamming_tc_range needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(q, flush=True)
    N, M = 2048, 65536
    X, y = T._history(N)
    Xt = T._one_hot(X)
    codes = T._grid(M)
    Xc = torch.as_tensor(T._one_hot(codes, np.float32), device="cuda")
    for S in args.s:
        l = S / T.ACTIVE
        f = H.fit(X, y, T._theta(l))
        mu, sd = T._posterior(f, codes)
        for acq in ("ei", "lcb"):
            e = GPEngine(0, kernel="rbf", acq=acq, length_scale=T.HMAP.length_scale(l), noise=1e-3 + H.ALPHA, var_mode="auto").record_stages()
            e.tell(Xt, y)
            b = e.ask(Xc)
            a = H.acquisition(mu, sd, float(np.min(y)), acq, 0.01, 1.96)
            i = int(np.argmax(a))
            short = float((a[i] - a[b.index]) / max(1.0, abs(a[i])))
            print(json.dumps(dict(S=S, acq=acq, tensor_cores=bool(e.stages()), held=bool(b.index == i or short <= 1e-9),
                                  shortfall=short, pick=b.index, oracle=i)), flush=True)
            e.close()


if __name__ == "__main__":
    main()
