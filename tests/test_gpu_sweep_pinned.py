"""The tensor-core sweep's branch-and-bound, pinned bit for bit: per case, SHA-256 of
  stages     every stage record (kbo_debug_record_stages): stage, acquisition, calibration rows, survivor count, the bits of E, Eμ,
             the raw maxima they came from and the lower bound, and the sorted survivor list where the count fits the stage's cap
             (atomics make the order of a list nondeterministic, and past the cap also which rows it holds);
  decisions  last_decisions(), last_rank_error() and last_rank_mu_error();
  ask        each suggestion: index and the bits of value, mu and std;
and the stages each case runs with their survivor counts (`path`), so a reader sees which branch of the sweep a case pins.

Together the cases reach every stage kind, each acquisition, one gp_hedge sweep (kbo_sweep_multi), the three-product redo of a
flat landscape and a history with D > 128 (FP64 K* kernel and the one-product cluster kernel: there is no tensor-core K* above 128):
  ei, lcb            lazy-fit pruning decides
  pi                 lazy-fit pruning → full-fit pruning → interval test of the pruning survivors (float64 grid on the host)
  lcb-full-fit       lazy_inverse=False: the full-fit pruning pass first
  ei-no-prefix       rank_prefix=0: the interval test over the grid
  pi-three-product   tc_fast=False: the three-product window
  gp-hedge           EI, LCB and PI over one posterior
  flat-ei            ¾ of the trials in a ball of radius 0.03, y = 10‖x − x₀‖² + noise: every pruning stage keeps the whole grid,
                     the interval test overflows and the sweep is redone with three products
  d160-pi            N = 2048, D = 160

The digests were recorded on one NVIDIA H100 80GB HBM3 at a 700 W power limit (driver 580.159.03), with the library as it was
before the sweep's single-CTA variance kernel and its refinement switch were removed and its duplicated pruning-stage kernels
merged.  They were the same in two separate processes.
"""
import hashlib
import json
import struct
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CAPS = {"lazy-prune": 16384, "prune": 16384, "prune-interval": 4096, "interval": 4096, "window": 4096}
M = 131072
CASES = {
    "ei": dict(N=4096, D=32, acq="ei"),
    "lcb": dict(N=4096, D=32, acq="lcb"),
    "pi": dict(N=4096, D=32, acq="pi", grid="host64"),
    "lcb-full-fit": dict(N=4096, D=32, acq="lcb", kw=dict(lazy_inverse=False)),
    "ei-no-prefix": dict(N=4096, D=32, acq="ei", kw=dict(rank_prefix=0)),
    "pi-three-product": dict(N=4096, D=32, acq="pi", kw=dict(tc_fast=False)),
    "gp-hedge": dict(N=4096, D=32, acq=("ei", "lcb", "pi")),
    "flat-ei": dict(N=4096, D=4, acq="ei", flat=True),
    "d160-pi": dict(N=2048, D=160, acq="pi"),
}

PINNED = {
    "ei": dict(
        path="lazy-prune ei 1",
        stages="f50bfdfaf68686b983e5fdd9992a99e76626676e57c52052c877b58fc86e097a",
        decisions="51eed8a1869eba9b4d173e0610e3f14cedcc58626fd7c64d9fdf29874cac1da6",
        ask="f89d7a9ad9e660c4a028e1ca11b055cbe5ea85a3d61672f8bf5cf961af48926d",
    ),
    "lcb": dict(
        path="lazy-prune lcb 12",
        stages="e46b0ad3614fc7f7580bc048d52696281173204b23f5be7433cfecdead1901e6",
        decisions="f3236539b42238d8830bfb33cd67d305832ea024436646cc65414429b0eada83",
        ask="76d20a1123cf8a9856a299e16a3f21d7a530dd9876f3bbbe3c772aa28a1b5bea",
    ),
    "pi": dict(
        path="lazy-prune pi 780 > prune pi 780 > prune-interval pi 55",
        stages="77a816e3852810f1062a8d55f60244d2493c0f9ac1ae187074c8e19ff55d05bf",
        decisions="52fd511d07d1d8a9953a88f9e7d892b1fb50b6a5cee7cbb9801d5f3764cb86a8",
        ask="cbb4041a5018916a74b1ef9c5d6d6db56164633663f23ecd523dd33c24ce4d89",
    ),
    "lcb-full-fit": dict(
        path="prune lcb 14 > prune-interval lcb 1",
        stages="e0acaf3029f1ec2f4867d7e31113e7fc0a4c25b6d787cc3d00579778dc85b952",
        decisions="0f3adb9c04e7c7e33fbee524a0c49919c0de489ca6b6199135cb45e99c48560b",
        ask="61e285553ee9a682c5522fe47d4812f47fad52ccb0c245cee8a70bf4c617d5e3",
    ),
    "ei-no-prefix": dict(
        path="interval ei 1",
        stages="d58830a354dfc3013aabae03573cd4649ca29246d53f70ac4b13bb5c959fb0d2",
        decisions="5af10d8cded72e1ac260be88b62e09626f4cef896173ac8719501be67ff63a42",
        ask="9704b192f1863441c2be2da254f89f3902a94fbdea687da202f03d0b570f35a0",
    ),
    "pi-three-product": dict(
        path="window pi 82",
        stages="26a9d4dc983c45b41fa5686a5373bf1fefeefe396c568eec0b5543c4257c7f4c",
        decisions="909921f19de748a170320fc695fba20bebfe3983bf38b658d8e5a32baefcefb2",
        ask="9c11effa921ea80fc7b7063816b930945da9060e26ef198466ac72576cb18ae2",
    ),
    "gp-hedge": dict(
        path="lazy-prune ei 1 > lazy-prune lcb 12 > lazy-prune pi 780 > prune pi 780 > prune-interval pi 55",
        stages="0ad6ba29e1e1305fd5172d7f8eaea62fb73452f5b3295aa5a4ac4d1ea3c667c1",
        decisions="63f92c6b5bb16ecbe4cb3f22102446cc7f698a764133a7a040bbb2fc1f091124",
        ask="bcd51e87aab8754d727cfd86eba55d286cde6c2a9b3c95ef8c79655755f735f4",
    ),
    "flat-ei": dict(
        path="lazy-prune ei 131072 > prune ei 131072 > interval ei 131072 > window ei 4",
        stages="b9fffc1922280e424469d35f1a15670c653678b3dccf0932d41d5edaeb7c3382",
        decisions="a24ab13b706bbc7c7fb869a3e7d6b2ed7a9a55189f1d6cad53626a0e64cd3ac2",
        ask="791c357e20c5503292c1c46d9131177138f94871fac9d3f37ae088a00650606e",
    ),
    "d160-pi": dict(
        path="interval pi 1",
        stages="14d656e07c62fbeb08f609c4328eac0bfcafac65e62564b5e85118d80d06b513",
        decisions="f45c6f5e2d6c462e77ae1eecc72a6d423d7fa8f9995fd196273b21f463ac2798",
        ask="db87d0c89e09ab95c236b4ae6eea25361dba57549cbcd485d21929cd488b701e",
    ),
}


def _data(c):
    from kubeflow_b200 import workload as W
    from oracle import gp_oracle as O
    from tests import _grid_cases as G
    N, D = c["N"], c["D"]
    X, y, _ = O.synthetic(N, 1, D)
    Xc = W.candidates(M, D, dtype=np.float64 if c.get("grid") == "host64" else np.float32)
    if c.get("flat"):   # the construction of _grid_cases' converged-d4, at an eighth of its grid
        r = np.random.default_rng(23)
        x0 = 0.2 + 0.6 * r.random(D)
        k = 3 * N // 4
        X[:k] = x0 + G._ball(r, k, D, 0.03)
        y = 10.0 * ((X - x0) ** 2).sum(1) + 0.1 * r.standard_normal(N)
        Xc[r.choice(M, M // 64, replace=False)] = (x0 + G._ball(r, M // 64, D, 0.06)).astype(Xc.dtype)
    return X, y, Xc, O.theta_of_record(D)


def _bits(*v):
    return struct.pack(f"<{len(v)}d", *v)


def run(name):
    """(path, digests) of one case on a fresh engine."""
    import torch
    from kubeflow_b200.gp import GPEngine
    c = CASES[name]
    X, y, Xc, th = _data(c)
    if c.get("grid") != "host64":
        Xc = torch.as_tensor(Xc, device="cuda")
    acqs = c["acq"] if isinstance(c["acq"], tuple) else (c["acq"],)
    e = GPEngine(0, kernel="matern52", acq=acqs[0], **th, **c.get("kw", {})).record_stages()
    e.tell(X, y)
    bests = e.ask_multi(Xc, list(acqs)) if len(acqs) > 1 else [e.ask(Xc)]
    recs = e.stages()
    h_st = hashlib.sha256()
    for s in recs:
        h_st.update(f"{s['stage']},{s['acq']},{s['cal_n']},{s['n']};".encode())
        h_st.update(_bits(s["E"], s["E_mu"], s["dvar_raw"], s["dmu_raw"], s["lb"]))
        if s["n"] <= CAPS[s["stage"]]:
            h_st.update(np.ascontiguousarray(s["survivors"], dtype="<i8").tobytes())
    h_dec = hashlib.sha256(repr(e.last_decisions()).encode() + _bits(e.last_rank_error(), e.last_rank_mu_error()))
    h_ask = hashlib.sha256()
    for b in bests:
        h_ask.update(struct.pack("<q", b.index) + _bits(b.value, b.mu, b.std))
    e.close()
    path = " > ".join(f"{s['stage']} {s['acq']} {s['n']}" for s in recs)
    return path, dict(stages=h_st.hexdigest(), decisions=h_dec.hexdigest(), ask=h_ask.hexdigest())


@pytest.mark.parametrize("name", list(CASES))
def test_sweep_matches_its_pinned_digests(name):
    path, got = run(name)
    want = PINNED[name]
    assert path == want["path"], name
    assert got == {k: v for k, v in want.items() if k != "path"}, name


if __name__ == "__main__":   # re-record: python -m tests.test_gpu_sweep_pinned [case ...]
    for name in sys.argv[1:] or CASES:
        path, d = run(name)
        print(json.dumps({name: dict(path=path, **d)}), flush=True)
