"""CPU: the servicer list ``server.main`` serves — every algorithm name Katib ships routes to a service, plain and SPMD — and,
over gloo with world size 2, an SPMD servicer answers ``grid`` and ``darts`` on rank 0 alone, without a broadcast."""
import json
import os

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from kubeflow_b200.suggestion.server import services
from kubeflow_b200.suggestion.service import DispatchService

KATIB_ALGORITHMS = ("bayesianoptimization", "tpe", "multivariate-tpe", "cmaes", "enas", "hyperband", "pbt", "random", "sobol",
                    "grid", "darts")


def test_every_katib_algorithm_routes():
    from tests.test_grpc_service import make_experiment
    for shard in (False, True):
        d = DispatchService(services({"device": 0}, shard=shard))
        assert sorted(d._by_name) == sorted(KATIB_ALGORITHMS)
        for name in KATIB_ALGORITHMS:
            assert name in d._pick(make_experiment(name)).algorithm_names
        assert {n for n, s in d._by_name.items() if getattr(s, "engine_defaults", {}).get("shard")} == (
            {"bayesianoptimization", "tpe", "multivariate-tpe"} if shard else set())


def _worker(rank, world, pg_port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(pg_port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import grpc
    from kubeflow_b200.suggestion import api_pb as api
    from kubeflow_b200.suggestion.server import SuggestionStub, serve
    from kubeflow_b200.suggestion.spmd import SpmdServicer
    from tests.test_darts_service import make_experiment as darts_experiment
    from tests.test_grid_service import make_experiment as grid_experiment
    spmd = SpmdServicer(DispatchService(services({"device": 0}, shard=True)))
    result = {"rank": rank}
    if rank == 0:
        server, port = serve(spmd, port=0, host="127.0.0.1")
        ch = grpc.insecure_channel(f"127.0.0.1:{port}")
        stub = SuggestionStub(ch)
        replies = {}
        for name, exp in (("grid", grid_experiment(settings={"random_state": 1}, name="spmd-grid")),
                          ("darts", darts_experiment(name="spmd-darts"))):
            stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
            rep = stub.GetSuggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=3))
            replies[name] = [[a.name for a in pa.assignments] for pa in rep.parameter_assignments]
        result.update(replies=replies, calls_before_stop=spmd.calls)
        ch.close()
        server.stop(0)
        spmd.stop()
    else:
        spmd.worker_loop()
    result["calls"] = spmd.calls
    q.put(result)
    dist.barrier()
    dist.destroy_process_group()


def test_spmd_answers_grid_and_darts_on_rank_0_without_a_broadcast():
    from tests.test_spmd_gloo import _free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    out = sorted([q.get(timeout=300) for _ in ps], key=lambda d: d["rank"])
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    r0, r1 = out
    assert r0["calls_before_stop"] == r0["calls"] == r1["calls"] == 0
    assert r0["replies"] == {"grid": [["lr", "layers", "opt"]] * 3, "darts": [["algorithm-settings", "search-space", "num-layers"]] * 3}


def test_the_katib_config_patch_routes_every_algorithm_to_the_image():
    yaml = pytest.importorskip("yaml")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "deploy", "katib-config-patch.yaml")) as f:
        routes = json.loads(yaml.safe_load(f)["data"]["suggestion"])
    assert sorted(routes) == sorted(KATIB_ALGORITHMS)
    host_only = {"hyperband", "pbt", "random", "sobol", "grid", "darts"}
    assert {n for n, r in routes.items() if "resources" not in r} == host_only
