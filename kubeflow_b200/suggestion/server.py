"""gRPC server for ``api.v1.beta1.Suggestion`` on port 6789 (Katib's DefaultSuggestionPort), generic handlers —
no generated stubs needed.  Registers the upstream service name ``api.v1.beta1.Suggestion`` and the alias
``api.v1.beta1.SuggestionService`` (BASELINE.json's spelling), plus a hand-registered ``grpc.health.v1.Health/Check``
(grpc_health is not in this image) that Katib's readiness probe calls.

    python -m kubeflow_b200.suggestion.server --port 6789
"""
from __future__ import annotations

import argparse
import logging
from concurrent import futures

import grpc

from . import api_pb as api
from .ingest import LazyRequest

DEFAULT_PORT = 6789
SERVICE_NAMES = (f"{api.PACKAGE}.Suggestion", f"{api.PACKAGE}.SuggestionService")
_HEALTH_SERVING = b"\x08\x01"   # HealthCheckResponse{status: SERVING}  (field 1 varint 1)


def add_suggestion_servicer(servicer, server: grpc.Server):
    handlers = {
        "GetSuggestions": grpc.unary_unary_rpc_method_handler(
            servicer.GetSuggestions, request_deserializer=LazyRequest.FromString,   # wire bytes kept: see ingest.py
            response_serializer=lambda m: m.SerializeToString()),
        "ValidateAlgorithmSettings": grpc.unary_unary_rpc_method_handler(
            servicer.ValidateAlgorithmSettings, request_deserializer=api.ValidateAlgorithmSettingsRequest.FromString,
            response_serializer=lambda m: m.SerializeToString()),
    }
    for name in SERVICE_NAMES:
        server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(name, handlers),))
    health = {"Check": grpc.unary_unary_rpc_method_handler(lambda req, ctx: _HEALTH_SERVING, request_deserializer=lambda b: b,
                                                           response_serializer=lambda b: b)}
    server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler("grpc.health.v1.Health", health),))


def serve(servicer, port: int = DEFAULT_PORT, max_workers: int = 4, host: str = "0.0.0.0"):
    # a cfg3-sized request (8192 trials × 32 parameters as strings) is ~11 MB: lift gRPC's 4 MB default
    server = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers),
                         options=[("grpc.max_receive_message_length", 1 << 28), ("grpc.max_send_message_length", 1 << 28)])
    add_suggestion_servicer(servicer, server)
    bound = server.add_insecure_port(f"{host}:{port}")
    server.start()
    return server, bound


class SuggestionStub:
    """Client-side stub (what katib-controller's suggestion client does), used by the tests and INTEGRATION.md."""

    def __init__(self, channel: grpc.Channel, service_name: str = SERVICE_NAMES[0]):
        self.GetSuggestions = channel.unary_unary(f"/{service_name}/GetSuggestions",
                                                  request_serializer=lambda m: m.SerializeToString(),
                                                  response_deserializer=api.GetSuggestionsReply.FromString)
        self.ValidateAlgorithmSettings = channel.unary_unary(f"/{service_name}/ValidateAlgorithmSettings",
                                                             request_serializer=lambda m: m.SerializeToString(),
                                                             response_deserializer=api.ValidateAlgorithmSettingsReply.FromString)
        self.HealthCheck = channel.unary_unary("/grpc.health.v1.Health/Check", request_serializer=lambda b: b,
                                               response_deserializer=lambda b: b)


def services(dev: dict, shard: bool = False) -> list:
    """The servicers ``main`` routes to, one per algorithm name Katib ships; ``dev`` holds the engine defaults (``device``), and
    ``shard`` makes the algorithms that shard their candidates over the ranks of an SPMD run (suggestion/spmd.py) do so."""
    from .cmaes_service import CmaesService
    from .darts_service import DartsService
    from .enas_service import EnasService
    from .grid_service import GridService
    from .hyperband import HyperbandService
    from .mvtpe_service import MultivariateTpeService
    from .pbt_service import PbtService
    from .service import RandomService, SkoptService, SobolService
    from .tpe_service import TpeService
    sharded = {**dev, "shard": True} if shard else dev
    return [SkoptService(sharded), RandomService(), SobolService(), CmaesService(dev), TpeService(sharded),
            MultivariateTpeService(sharded), EnasService(dev), HyperbandService(), PbtService(), GridService(), DartsService()]


def main():
    from .service import DispatchService
    ap = argparse.ArgumentParser()
    ap.add_argument("--port", type=int, default=DEFAULT_PORT)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--spmd", action="store_true",
                    help="one process per GPU under torchrun: rank 0 serves gRPC, every request runs on all ranks with the candidate "
                         "grid sharded (suggestion/spmd.py)")
    args = ap.parse_args()
    logging.basicConfig(level=logging.INFO)
    if args.spmd:
        import os
        import torch
        import torch.distributed as dist
        from .spmd import SpmdServicer
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        spmd = SpmdServicer(DispatchService(services({"device": local}, shard=True)))
        if dist.get_rank() == 0:
            server, port = serve(spmd, args.port)
            logging.info("api.v1.beta1.Suggestion listening on :%d, %d ranks", port, dist.get_world_size())
            try:
                server.wait_for_termination()
            finally:
                spmd.stop()
        else:
            spmd.worker_loop()
        dist.destroy_process_group()
        return
    server, port = serve(DispatchService(services({"device": args.device})), args.port)
    logging.info("api.v1.beta1.Suggestion listening on :%d", port)
    server.wait_for_termination()


if __name__ == "__main__":
    main()
