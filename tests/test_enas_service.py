"""CPU: the ``enas`` service without a device — search-space expansion, the reply strings for a fixed arc, every settings and
``nas_config`` refusal and the engine limits over a real gRPC server, and the reward filter (the controller itself is tested
on the GPU in tests/test_gpu_enas.py)."""
import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.enas_service import (DEFAULTS, EnasService, expand_operations, reply_assignments, reward_of,
                                                   validate_enas_settings)
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, RandomService

# two operations expanding to 4 + 2 = 6 operation ids
OPERATIONS = (("convolution", (("filter_size", api.CATEGORICAL, None, None, None, ("3", "5")), ("num_filter", api.INT, "32", "64", "32", ()))),
              ("reduction", (("reduction_type", api.CATEGORICAL, None, None, None, ("max_pooling", "avg_pooling")),)))


def make_experiment(settings=None, name="enas-1", num_layers=5, operations=OPERATIONS, input_sizes=(32, 32, 3), output_sizes=(10,),
                    algorithm="enas"):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MAXIMIZE
    e.spec.objective.objective_metric_name = "accuracy"
    e.spec.algorithm.algorithm_name = algorithm
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    gc = e.spec.nas_config.graph_config
    gc.num_layers = num_layers
    gc.input_sizes.extend(input_sizes)
    gc.output_sizes.extend(output_sizes)
    for op_type, specs in operations:
        op = e.spec.nas_config.operations.operation.add()
        op.operation_type = op_type
        for pname, ptype, lo, hi, step, lst in specs:
            p = op.parameter_specs.parameters.add()
            p.name, p.parameter_type = pname, ptype
            if lo is not None:
                p.feasible_space.min = lo
            if hi is not None:
                p.feasible_space.max = hi
            if step is not None:
                p.feasible_space.step = step
            p.feasible_space.list.extend(lst)
    return e


@pytest.fixture(scope="module")
def stub():
    svc = EnasService()
    server, port = serve(DispatchService([RandomService(), svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


def _refused(s, exp, needle):
    with pytest.raises(grpc.RpcError) as ei:
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and needle in ei.value.details(), ei.value.details()


def test_expansion_int_double_categorical_and_product_order():
    ops = (("conv", (("k", api.INT, "1", "7", "3", ()), ("act", api.CATEGORICAL, None, None, None, ("relu", "tanh")))),
           ("drop", (("rate", api.DOUBLE, "0.1", "0.5", "0.15", ()),)))
    out = expand_operations(make_experiment(operations=ops).spec.nas_config.operations.operation)
    assert [o["opt_id"] for o in out] == list(range(9))
    assert [o["opt_params"] for o in out[:6]] == [{"k": k, "act": a} for k in (1, 4, 7) for a in ("relu", "tanh")]   # last spec fastest
    assert all(o["opt_type"] == "conv" for o in out[:6]) and all(o["opt_type"] == "drop" for o in out[6:])
    assert [o["opt_params"]["rate"] for o in out[6:]] == pytest.approx([0.1, 0.25, 0.4])      # arange's 0.55 > max is dropped
    assert all(type(o["opt_params"]["k"]) is int for o in out[:6]) and all(type(o["opt_params"]["rate"]) is float for o in out[6:])


def test_reply_strings_for_a_fixed_arc():
    ops = expand_operations(make_experiment().spec.nas_config.operations.operation)
    arc = [2, 5, 0, 2, 1, 1]                                # layers: [2], [5, 0], [2, 1, 1]
    a, n = reply_assignments(arc, 3, [32, 32, 3], [10], ops)
    assert a.name == "architecture" and a.value == "[[2], [5, 0], [2, 1, 1]]"
    assert n.name == "nn_config"
    assert n.value == ("{'num_layers': 3, 'input_sizes': [32, 32, 3], 'output_sizes': [10], 'embedding': "
                       "{'2': {'opt_id': 2, 'opt_type': 'convolution', 'opt_params': {'filter_size': '5', 'num_filter': 32}}, "
                       "'5': {'opt_id': 5, 'opt_type': 'reduction', 'opt_params': {'reduction_type': 'avg_pooling'}}}}")


@pytest.mark.parametrize("name,value", [
    ("controller_hidden_size", 0), ("controller_hidden_size", "x"), ("controller_hidden_size", "None"), ("controller_temperature", 0),
    ("controller_temperature", -1), ("controller_tanh_const", 0), ("controller_entropy_weight", -0.1), ("controller_baseline_decay", 1.5),
    ("controller_baseline_decay", -0.1), ("controller_learning_rate", 0), ("controller_learning_rate", 1.5), ("controller_skip_target", 0),
    ("controller_skip_target", 1), ("controller_skip_weight", -1), ("controller_train_steps", 0), ("controller_log_every_steps", 0),
    ("controller_log_every_steps", "1.5"), ("random_state", -1), ("device", -1), ("bogus", 1)])
def test_bad_settings_are_invalid_argument_naming_the_setting(stub, name, value):
    _refused(stub[0], make_experiment({name: value}), name)


def test_good_settings_and_defaults(stub):
    ok = {"controller_hidden_size": 128, "controller_temperature": "None", "controller_tanh_const": "None", "controller_entropy_weight": "None",
          "controller_skip_weight": "None", "controller_baseline_decay": 0, "controller_learning_rate": 1, "controller_skip_target": 0.5,
          "controller_train_steps": 10000, "controller_log_every_steps": 1, "random_state": 3, "device": 0}
    stub[0].ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(ok)))
    got = validate_enas_settings({k: str(v) for k, v in ok.items()})
    assert got["controller_temperature"] is None and got["controller_skip_weight"] is None and got["controller_train_steps"] == 10000
    assert validate_enas_settings({}) == DEFAULTS


@pytest.mark.parametrize("kw,needle", [
    (dict(num_layers=0), "num_layers"), (dict(input_sizes=()), "input_sizes"), (dict(output_sizes=()), "output_sizes"),
    (dict(operations=()), "at least one operation"),
    (dict(operations=(("", (("a", api.CATEGORICAL, None, None, None, ("x",)),)),)), "operation_type"),
    (dict(operations=(("conv", ()),)), "at least one parameter spec"),
    (dict(operations=(("conv", (("k", api.INT, "1", "7", None, ()),)),)), "min, max and step"),
    (dict(operations=(("conv", (("k", api.INT, "1", None, "1", ()),)),)), "min, max and step"),
    (dict(operations=(("conv", (("k", api.INT, "7", "1", "1", ()),)),)), "min <= max"),
    (dict(operations=(("conv", (("k", api.DOUBLE, "0", "1", "-0.5", ()),)),)), "step > 0"),
    (dict(operations=(("conv", (("k", api.CATEGORICAL, None, None, None, ()),)),)), "non-empty list"),
    (dict(operations=(("conv", (("k", api.DISCRETE, None, None, None, ("1", "2")),)),)), "only INT, DOUBLE and CATEGORICAL"),
])
def test_nas_config_refusals(stub, kw, needle):
    _refused(stub[0], make_experiment(**kw), needle)


def test_engine_limits(stub):
    s = stub[0]
    _refused(s, make_experiment(num_layers=65), "limit of 64")
    _refused(s, make_experiment({"controller_hidden_size": 129}), "limit of 128")
    _refused(s, make_experiment({"controller_train_steps": 10001}), "limit of 10000")
    wide = (("conv", (("a", api.INT, "1", "64", "1", ()), ("b", api.INT, "1", "65", "1", ()))),)
    _refused(s, make_experiment(operations=wide), "limit of 4096")
    edge = (("conv", (("a", api.INT, "1", "64", "1", ()), ("b", api.INT, "1", "64", "1", ()))),)
    s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(operations=edge)))   # exactly 4096
    with pytest.raises(grpc.RpcError) as ei:
        s.GetSuggestions(api.GetSuggestionsRequest(experiment=make_experiment(name="enas-big-k"), current_request_number=1025))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and "limit of 1024" in ei.value.details()


def test_zero_arcs_reply_empty_without_a_controller(stub):
    s, svc = stub
    rep = s.GetSuggestions(api.GetSuggestionsRequest(experiment=make_experiment(name="enas-zero"), current_request_number=0))
    assert len(rep.parameter_assignments) == 0 and "enas-zero" not in svc._exps


def test_reward_is_the_mean_over_succeeded_trials_of_the_named_metric():
    req = api.GetSuggestionsRequest()
    for name, cond, metrics in (("a", api.SUCCEEDED, (("loss", "9"), ("accuracy", "0.5"))), ("b", api.SUCCEEDED, (("accuracy", "0.7"),)),
                                ("c", api.EARLYSTOPPED, (("accuracy", "100"),)), ("d", api.FAILED, (("accuracy", "-100"),)),
                                ("e", api.TRIAL_CONDITIONS.index("RUNNING"), (("accuracy", "50"),)), ("f", api.SUCCEEDED, (("loss", "3"),))):
        t = req.trials.add()
        t.name, t.status.condition = name, cond
        for k, v in metrics:
            m = t.status.observation.metrics.add()
            m.name, m.value = k, v
    assert reward_of(req.trials, "accuracy") == pytest.approx(0.6)
    assert reward_of(req.trials, "loss") == pytest.approx(6.0)
    assert reward_of(req.trials[2:5], "accuracy") is None


def test_routing_through_dispatch(stub):
    _refused(stub[0], make_experiment(algorithm="enas2"), "enas2")


@pytest.mark.parametrize("ops", [OPERATIONS,
                                 (("conv", (("k", api.INT, "1", "7", "3", ()), ("act", api.CATEGORICAL, None, None, None, ("relu", "tanh")),
                                            ("drop", api.DOUBLE, "0.1", "0.5", "0.15", ()))),
                                  ("pool", (("size", api.INT, "2", "2", "1", ()),)),
                                  ("dense", (("rate", api.DOUBLE, "0.0", "1.0", "0.25", ()), ("units", api.INT, "8", "32", "8", ()))))])
def test_service_expansion_and_replies_equal_the_oracle_restatement(ops):
    import numpy as np
    from oracle import enas_oracle as O
    exp = make_experiment(operations=ops)
    mine = expand_operations(exp.spec.nas_config.operations.operation)
    ref = O.expand(exp.spec.nas_config.operations.operation)
    assert [(o["opt_type"], o["opt_params"]) for o in mine] == ref
    assert [[type(v) for v in o["opt_params"].values()] for o in mine] == [[type(v) for v in p.values()] for _, p in ref]
    rng = np.random.default_rng(len(ref))
    for L in (1, 2, 5):
        arc = [int(rng.integers(len(ref))) if j == 0 else int(rng.integers(2)) for l in range(L) for j in range(l + 1)]
        a, n = reply_assignments(arc, L, [32, 32, 3], [10], mine)
        assert (a.value, n.value) == O.reply_strings(arc, L, [32, 32, 3], [10], ref)
