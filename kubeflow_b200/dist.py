"""Multi-GPU plumbing for the sharded candidate grid (SURVEY.md §8(e)).

One process per GPU.  Rank r sweeps rows [r·M/R, (r+1)·M/R) of the grid with ``global_offset`` set, so every
rank's Best carries a GLOBAL index; the only exchange step is the argmax: one all-gather of (value, index, mu, std)
per rank, then every rank picks the maximum value / lowest index — i.e. exactly ``np.argmin(-values)`` (first maximal
index) over the concatenated grid.  32 bytes per rank over NCCL/NVLink; latency only.
Works with the ``nccl`` backend (CUDA tensors) and with ``gloo`` (CPU tensors; used by the CPU tests).
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from .gp import Best

def shard_rows(M: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous row block [lo, hi) of an M-row grid owned by `rank` (first M % world ranks get one extra)."""
    base, rem = divmod(M, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class RankFailure(RuntimeError):
    """A rank's local sweep failed; raised on EVERY rank after the exchange so nobody is left waiting in a collective."""


def global_argmax(best: Best | list[Best] | None, group=None, device=None, failed: str | None = None, n: int | None = None):
    """Combine per-rank Bests into the global first-index argmax with ONE collective: an all-gather of 5 doubles per rank
    (value, index, mu, std, failed flag); every rank then takes the maximum value, lowest global index among equals —
    exactly ``np.argmin(-values)`` over the concatenated grid.  Indices up to 2^53 are exact in a double.
    ``best`` may also be a list of Bests — one per acquisition of a multi-acquisition sweep, in the same order on every
    rank — and a list of global Bests is returned, still from ONE all-gather (5 doubles per entry and rank).  ``n``: the
    list's length, needed when this rank has no list to give (``failed``).
    ``failed``: a rank whose local sweep raised still JOINS the collective (with −inf and the flag set) and all ranks raise
    ``RankFailure`` together — a rank-local CUDA / not-PD error must not leave the others blocked in the all-gather."""
    multi = isinstance(best, list) or n is not None
    k = (len(best) if isinstance(best, list) else int(n)) if multi else 1
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        if failed:
            raise RankFailure(failed)
        return best
    world = dist.get_world_size(group)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    if failed or best is None:
        mine = torch.tensor([float("-inf"), float(2 ** 52), 0.0, 0.0, 1.0] * k, dtype=torch.float64, device=device)
    else:
        rows = []
        for b in (best if multi else [best]):
            v = b.value if b.value == b.value else float("-inf")   # NaN never wins
            rows += [v, float(b.index), b.mu, b.std, 0.0]
        mine = torch.tensor(rows, dtype=torch.float64, device=device)
    allv = torch.empty(world * 5 * k, dtype=torch.float64, device=device)
    dist.all_gather_into_tensor(allv, mine, group=group)
    table = allv.view(world, k, 5).cpu().tolist()
    bad = [r for r, rk in enumerate(table) if any(row[4] != 0.0 for row in rk)]
    if bad:
        raise RankFailure(f"local sweep failed on rank(s) {bad}" + (f": {failed}" if failed else ""))
    out = []
    for j in range(k):
        win = max((table[r][j] for r in range(world)), key=lambda r: (r[0], -r[1]))
        out.append(Best(float(win[0]), int(win[1]), float(win[2]), float(win[3])))
    return out if multi else out[0]


def rank0_seed() -> int:
    """A seed drawn from fresh entropy on rank 0 and broadcast: every rank of the default process group gets the same one."""
    import numpy as np
    box = [int(np.random.default_rng().integers(1 << 62))]
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast_object_list(box, src=0)
    return box[0]


def sharded_ask(shard_ask, pick, n_candidates: int, rows: int, device):
    """An ask over candidates sharded by index (``tpe`` / ``multivariate-tpe``): this rank's ``shard_ask(lo, hi)`` returns
    its (FP64 value, global index) winner per row (NumPy arrays of ``rows``); one ``global_argmax`` over the rows gives
    every rank the first index of the global maximum, and ``pick(indices)`` regenerates those candidates locally, so no row
    has to be broadcast.  A rank whose shard ask raises still joins the exchange and every rank raises ``RankFailure``.
    An empty shard's (-inf, n_candidates) entries are ordinary entries that never win."""
    lo, hi = shard_rows(n_candidates, dist.get_rank(), dist.get_world_size())
    bests, failed = None, None
    try:
        val, idx = shard_ask(lo, hi)
        bests = [Best(float(v), int(i), 0.0, 0.0) for v, i in zip(val.ravel().tolist(), idx.ravel().tolist())]
    except Exception as e:  # noqa: BLE001 — every rank raises RankFailure in the exchange, none is left waiting
        failed = f"{type(e).__name__}: {e}"
    bests = global_argmax(bests, device=device, failed=failed, n=rows)
    return pick([b.index for b in bests])
