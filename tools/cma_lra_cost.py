"""One JSON line: what CMA-ES with learning-rate adaptation costs on the GPU.

* ask + tell per generation at (D, λ) = (10, 10), (128, 18) and (128, 4096), without and with the adaptation:
  `kbo_cma_run_synthetic` (device fitness, CUDA events around the whole run), median of 5 runs of 200 generations after a
  20-generation warm-up.  The two variants alternate, each in its own instance.
* cma_lra_prep_kernel's, cma_lra_kernel's and cma_lra_finish_kernel's own time: torch.profiler with CUDA activities over
  200 generations, mean per launch.
The card, its power limit and max SM clock are read in the same run."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np

from tools.cma_restart_cost import card

KERNELS = ("cma_lra_prep_kernel", "cma_lra_kernel", "cma_lra_finish_kernel")


def kernel_ms(prof, name):
    ev = [e for e in prof.key_averages() if name + "(" in e.key or e.key == name]
    if not ev:
        return None
    t = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
    return t / ev[0].count / 1e3


def main():
    import torch
    from kubeflow_b200.cmaes import CmaEs
    out = card()
    for D, lam, fn in ((10, 10, "sphere"), (128, 18, "rastrigin"), (128, 4096, "rastrigin")):
        es = {}
        for variant in ("plain", "lra"):
            es[variant] = CmaEs(np.full(D, 3.0), 2.0, popsize=lam, seed=7)
            if variant == "lra":
                es[variant].set_lr_adapt(True)
            es[variant].run_synthetic(fn, 20)
        ms = {"plain": [], "lra": []}
        for _ in range(5):
            for variant in ("plain", "lra"):
                ms[variant].append(es[variant].run_synthetic(fn, 200)["elapsed_ms"] / 200)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            es["lra"].run_synthetic(fn, 200)
            torch.cuda.synchronize()
        res = {}
        for variant, v in ms.items():
            v = sorted(v)
            res[variant] = dict(ask_tell_ms_per_generation=v[len(v) // 2], ask_tell_ms_min=v[0], ask_tell_ms_max=v[-1])
        for k in KERNELS:
            res[f"{k}_ms"] = kernel_ms(prof, k)
        res["eta_after_240_generations"] = [es["lra"].lr_state()[k] for k in ("eta_mean", "eta_Sigma")]
        for e in es.values():
            e.close()
        out[f"d{D}_pop{lam}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
