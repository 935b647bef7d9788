"""One JSON line: the ENAS controller on the GPU — one train call of 50 REINFORCE steps and one sample call of k ∈ {1, 16, 256}
arcs (CUDA-event times, medians after warm-up) at (L, H, n_ops) ∈ {(8, 64, 78), (12, 64, 6), (24, 128, 1024)}, and the time per
dependent LSTM cell (a step runs 4·L of them: 2·L forward, 2·L backward).  In the same run, on the host's cores, two
restatements of the same 50 steps (neither is upstream's TF graph): the FP64 NumPy oracle and an FP32 torch-CPU controller
with autograd and torch's Adam.  The card, its power limit and max SM clock are read in the same run."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from kubeflow_b200.enas import DEFAULT_SETTINGS, EnasController

SHAPES = ((8, 64, 78), (12, 64, 6), (24, 128, 1024))
STEPS = 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, pl, clk = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=float(clk))


def torch_cpu_steps(L, H, n_ops, steps, st=DEFAULT_SETTINGS):
    """An FP32 torch-CPU restatement of `steps` REINFORCE steps (sample, forward, autograd backward, Adam); seconds."""
    g = torch.Generator().manual_seed(0)
    u = lambda *s: (torch.rand(*s, generator=g) * 0.2 - 0.1).requires_grad_()
    W, ge, we, ws, w1, w2, v = u(2 * H, 4 * H), u(1, H), u(n_ops, H), u(H, n_ops), u(H, H), u(H, H), u(H, 1)
    opt = torch.optim.Adam([W, ge, we, ws, w1, w2, v], lr=st["learning_rate"], betas=(0.0, 0.999), eps=1e-3)
    tgt = torch.tensor([1 - st["skip_target"], st["skip_target"]])
    shp = lambda z: st["tanh_const"] * torch.tanh(z / st["temperature"])
    baseline = 0.0
    t0 = time.perf_counter()
    for _ in range(steps):
        c = h = torch.zeros(H)
        x = ge[0]
        nll, kls, anchors, aw = 0.0, [], [], []

        def cell(x, c, h):
            z = torch.cat([x, h]) @ W
            i, f, o, gg = torch.sigmoid(z[:H]), torch.sigmoid(z[H:2 * H]), torch.sigmoid(z[2 * H:3 * H]), torch.tanh(z[3 * H:])
            c = i * gg + f * c
            return c, o * torch.tanh(c)
        for l in range(L):
            c, h = cell(x, c, h)
            lp = torch.log_softmax(shp(h @ ws), 0)
            op = int(torch.multinomial(lp.exp().detach(), 1, generator=g))
            nll = nll - lp[op]
            c, h = cell(we[op], c, h)
            if l > 0:
                q = (torch.tanh(torch.stack(aw) + h @ w2) @ v)[:, 0]
                s = shp(torch.stack([-q, q], 1))
                lp2 = torch.log_softmax(s, 1)
                sk = torch.multinomial(lp2.exp().detach(), 1, generator=g)[:, 0]
                nll = nll - lp2.gather(1, sk[:, None]).sum()
                gs = torch.sigmoid(s)
                kls.append((gs * torch.log(gs / tgt)).sum())
                x = (sk.float()[:, None] * torch.stack(anchors)).sum(0) / (1.0 + sk.sum())
            else:
                x = ge[0]
            anchors.append(h)
            aw.append(h @ w1)
        r = 0.5
        baseline -= (1 - st["baseline_decay"]) * (baseline - r)
        loss = nll * (r - baseline) + (st["skip_weight"] * torch.stack(kls).mean() if kls else 0.0)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return time.perf_counter() - t0


def oracle_steps(L, H, n_ops, steps):
    from oracle import enas_oracle as O
    st = O.settings()
    rng = np.random.default_rng(0)
    s = O.new_state(O.init_params(H, n_ops, rng))
    t0 = time.perf_counter()
    for _ in range(steps):
        O.train_step(s, L, st, 0.5, uniforms=rng.random(L * (L + 1) // 2))
    return time.perf_counter() - t0


def main():
    info = card()
    rows = []
    for L, H, n_ops in SHAPES:
        ctl = EnasController(L, H, n_ops, seed=1)
        ctl.sample(1)
        ctl.train(0.5, STEPS)                                   # warm-up
        tr = []
        for _ in range(5):
            ctl.train(0.5, STEPS)
            tr.append(ctl.last_timings()["train_ms"])
        smp = {}
        for k in (1, 16, 256):
            ctl.sample(k)
            ts = []
            for _ in range(5):
                ctl.sample(k)
                ts.append(ctl.last_timings()["sample_ms"])
            smp[str(k)] = float(np.median(ts))
        ctl.close()
        train_ms = float(np.median(tr))
        host_steps = STEPS if L * H < 2000 else 10                # the larger shape: 10 steps, scaled to 50
        rows.append(dict(L=L, H=H, n_ops=n_ops, train_50_steps_ms=train_ms, train_ms_range=[float(min(tr)), float(max(tr))],
                         us_per_dependent_cell=train_ms * 1e3 / (STEPS * 4 * L), sample_ms=smp,
                         numpy_fp64_oracle_50_steps_ms=oracle_steps(L, H, n_ops, host_steps) * 1e3 * STEPS / host_steps,
                         torch_cpu_fp32_50_steps_ms=torch_cpu_steps(L, H, n_ops, host_steps) * 1e3 * STEPS / host_steps,
                         host_steps_timed=host_steps))
    print(json.dumps(dict(info, host_threads=torch.get_num_threads(), cpu_count=os.cpu_count(), shapes=rows)))


if __name__ == "__main__":
    main()
