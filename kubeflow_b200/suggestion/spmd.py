"""One suggestion service over all GPUs of a node (SURVEY.md §8(e), BASELINE cfg5: one EI grid sharded over 8 GPUs).

``torchrun --nproc-per-node 8 -m kubeflow_b200.suggestion.server --spmd``: one process per GPU.  Rank 0 is the gRPC
endpoint Katib talks to; for every ``GetSuggestions`` it broadcasts the request's wire bytes and all ranks run the SAME
servicer call in lockstep — same trials told, same seed, same constant lies — so their optimizers stay identical without
any state exchange.  Inside the call the optimizer (``shard=True``) gives each rank ``n_points / world`` candidates, the
fit is replicated, and the only data-path collectives are the 32-byte all-gather of the per-rank argmax
(``dist.global_argmax``) and the broadcast of the winning row from its owner.  ``tpe`` and ``multivariate-tpe`` shard the
same way: each rank draws and scores its block of every point's candidates (keyed by their global index), one all-gather
of the per-rank (FP64 value, global index) winners decides, and every rank regenerates the winners itself
(``dist.sharded_ask``), so the replies are bit for bit those of one GPU.  Ranks > 0 sit in ``worker_loop``.
Calls are serialised on rank 0 (collectives need one order); ValidateAlgorithmSettings touches no GPU and stays on rank 0.
"""
from __future__ import annotations

import logging
import threading

import torch.distributed as dist

from .ingest import LazyRequest

logger = logging.getLogger(__name__)


class SpmdServicer:
    sharded_algorithms = ("", "bayesianoptimization", "tpe", "multivariate-tpe")

    def __init__(self, inner):
        if not dist.is_initialized():
            raise RuntimeError("SpmdServicer needs an initialised torch.distributed process group (launch with torchrun)")
        self.inner = inner
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self._lock = threading.Lock()
        self.calls = 0

    @staticmethod
    def _bcast(obj):
        box = [obj]
        dist.broadcast_object_list(box, src=0)
        return box[0]

    # -- rank 0: the gRPC-facing methods ---------------------------------------------------------------------------------
    def ValidateAlgorithmSettings(self, request, context):
        return self.inner.ValidateAlgorithmSettings(request, context)

    def GetSuggestions(self, request, context):
        if request.experiment.spec.algorithm.algorithm_name not in self.sharded_algorithms:
            return self.inner.GetSuggestions(request, context)      # nothing to shard (random, sobol, cmaes, enas, hyperband, pbt): rank 0 alone
        data = request._data if isinstance(request, LazyRequest) else request.SerializeToString()
        with self._lock:
            self._bcast(("GetSuggestions", data))
            self.calls += 1
            return self.inner.GetSuggestions(LazyRequest(data), context)

    def stop(self):
        with self._lock:
            self._bcast(("stop", b""))

    # -- ranks > 0 ---------------------------------------------------------------------------------------------------------
    def worker_loop(self):
        while True:
            cmd, data = self._bcast(None)
            if cmd == "stop":
                return
            self.calls += 1
            try:
                self.inner.get_suggestions(LazyRequest(data))
            except Exception as e:  # noqa: BLE001 — rank 0 meets the same error and reports it to the client
                logger.warning("rank %d: request failed like on rank 0: %s", self.rank, e)
