"""One JSON line: what CMA-ES with Margin costs on the GPU.

* ask + tell per generation at (D = 128, λ = 4096) and (D = 10, λ = 10), without and with the margin on half the
  dimensions (every other one: a 5-level table, a binary one, a 5001-level arithmetic range): `kbo_cma_run_synthetic`
  (device fitness, CUDA events around the whole run), median of 5 runs of 200 generations after a 20-generation warm-up.
  The two variants alternate, each in its own instance.
* cma_margin_kernel's and cma_x_margin_kernel's own time: torch.profiler with CUDA activities over 200 generations, mean
  per launch.
The card, its power limit and max SM clock are read in the same run."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np

from tools.cma_restart_cost import card


def dims(D):
    kinds = [np.linspace(0, 1, 5), np.array([0.0, 1.0]), (0.0, 1.0 / 5000, 5001)]
    return {j: kinds[(j // 2) % len(kinds)] for j in range(0, D, 2)}


def kernel_ms(prof, name):
    ev = [e for e in prof.key_averages() if name in e.key and (name != "cma_margin_kernel" or "x_margin" not in e.key)]
    if not ev:
        return None
    t = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
    return t / ev[0].count / 1e3


def main():
    import torch
    from kubeflow_b200.cmaes import CmaEs
    out = card()
    for D, lam, fn in ((128, 4096, "rastrigin"), (10, 10, "sphere")):
        es = {}
        for variant in ("plain", "margin"):
            es[variant] = CmaEs(np.full(D, 0.5), 1.0 / 6.0, popsize=lam, seed=7)
            if variant == "margin":
                es[variant].set_margin(dims(D))
            es[variant].run_synthetic(fn, 20)
        ms = {"plain": [], "margin": []}
        for _ in range(5):
            for variant in ("plain", "margin"):
                ms[variant].append(es[variant].run_synthetic(fn, 200)["elapsed_ms"] / 200)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            es["margin"].run_synthetic(fn, 200)
            torch.cuda.synchronize()
        res = {}
        for variant, v in ms.items():
            v = sorted(v)
            res[variant] = dict(ask_tell_ms_per_generation=v[len(v) // 2], ask_tell_ms_min=v[0], ask_tell_ms_max=v[-1])
        res["margin_kernel_ms"] = kernel_ms(prof, "cma_margin_kernel")
        res["x_margin_kernel_ms"] = kernel_ms(prof, "cma_x_margin_kernel")
        for e in es.values():
            e.close()
        out[f"d{D}_pop{lam}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
