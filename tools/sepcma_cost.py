"""One JSON line: what separable CMA-ES costs on the GPU, beside full CMA-ES where both run (D <= 128).

* ask + tell per generation at (D, λ) = (10, 10), (128, 18), (128, 4096), (1000, 24) and (4096, 28): a loop of ask,
  a Rastrigin fitness computed on the device with torch, and tell, timed by CUDA events around 200 generations; median of
  5 runs after a 20-generation warm-up.  Sep and full alternate, each in its own instance, with the same loop, so both
  figures include the same Python and torch overhead.  Full CMA-ES is also timed by `kbo_cma_run_synthetic` (device
  fitness, no Python in the loop), its figure of record.
* Each sep kernel's own time (sepcma_update_kernel, sepcma_finish_kernel, sepcma_should_stop_kernel and the shared
  cma_sort_kernel, cma_normal_kernel, cma_scale_kernel, cma_x_kernel): torch.profiler with CUDA activities over 200
  generations in a separate run, mean per launch.
The card, its power limit and max SM clock are read in the same run."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np

from tools.cma_lra_cost import kernel_ms
from tools.cma_restart_cost import card

SHAPES = ((10, 10), (128, 18), (128, 4096), (1000, 24), (4096, 28))
KERNELS = ("sepcma_update_kernel", "sepcma_finish_kernel", "sepcma_should_stop_kernel", "cma_sort_kernel", "cma_normal_kernel",
           "cma_scale_kernel", "cma_x_kernel")


def rastrigin(X):
    import torch
    return 10.0 * X.shape[1] + (X * X - 10.0 * torch.cos(2 * np.pi * X)).sum(1)


def loop_ms(es, gens):
    import torch
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(gens):
        es.tell(rastrigin(es.ask()))
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / gens


def main():
    import torch
    from kubeflow_b200.cmaes import CmaEs, SepCmaEs
    out = card()
    for D, lam in SHAPES:
        es = {"sep": SepCmaEs(np.full(D, 3.0), 2.0, popsize=lam, seed=7)}
        if D <= 128:
            es["full"] = CmaEs(np.full(D, 3.0), 2.0, popsize=lam, seed=7)
        for e in es.values():
            loop_ms(e, 20)
        ms = {k: [] for k in es}
        for _ in range(5):
            for k, e in es.items():
                ms[k].append(loop_ms(e, 200))
        res = {}
        for k, v in ms.items():
            v = sorted(v)
            res[k] = dict(ask_tell_ms_per_generation=v[len(v) // 2], ask_tell_ms_min=v[0], ask_tell_ms_max=v[-1])
        if "full" in es:
            es["full"].run_synthetic("rastrigin", 20)
            v = sorted(es["full"].run_synthetic("rastrigin", 200)["elapsed_ms"] / 200 for _ in range(5))
            res["full"]["device_loop_ms_per_generation"] = v[2]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            loop_ms(es["sep"], 200)
            torch.cuda.synchronize()
        res["sep_kernel_ms"] = {k: kernel_ms(prof, k) for k in KERNELS}
        res["sep_kernel_sum_ms"] = sum(v for v in res["sep_kernel_ms"].values() if v)
        res["sep_sigma_after"] = es["sep"].state()["sigma"]
        for e in es.values():
            e.close()
        out[f"d{D}_pop{lam}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
