"""CPU: Katib's ``darts`` algorithm through a real in-process gRPC server — the three reply strings for Katib's example DARTS
Experiment, with and without overriding settings; every refusal; replies of 0, 1 and 3 trials."""
import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.darts_service import DEFAULTS, DartsService, validate_darts_settings
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, RandomService

FILTERS = (("filter_size", api.CATEGORICAL, ("3", "5")),)
# Katib's example DARTS Experiment: separable and dilated convolutions 3/5, average and max pooling 3, skip_connection
OPERATIONS = (("separable_convolution", FILTERS), ("dilated_convolution", FILTERS),
              ("avg_pooling", (("filter_size", api.CATEGORICAL, ("3",)),)), ("max_pooling", (("filter_size", api.CATEGORICAL, ("3",)),)),
              ("skip_connection", ()))
SEARCH_SPACE = ("['separable_convolution_3x3', 'separable_convolution_5x5', 'dilated_convolution_3x3', 'dilated_convolution_5x5', "
                "'avg_pooling_3x3', 'max_pooling_3x3', 'skip_connection']")
DEFAULT_SETTINGS = ("{'num_epochs': 50, 'w_lr': 0.025, 'w_lr_min': 0.001, 'w_momentum': 0.9, 'w_weight_decay': 0.0003, "
                    "'w_grad_clip': 5.0, 'alpha_lr': 0.0003, 'alpha_weight_decay': 0.001, 'batch_size': 128, 'num_workers': 4, "
                    "'init_channels': 16, 'print_step': 50, 'num_nodes': 4, 'stem_multiplier': 3}")


def make_experiment(settings=None, name="darts-1", num_layers=8, operations=OPERATIONS, algorithm="darts"):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MAXIMIZE
    e.spec.objective.objective_metric_name = "Best-Genotype"
    e.spec.algorithm.algorithm_name = algorithm
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    e.spec.nas_config.graph_config.num_layers = num_layers
    for op_type, specs in operations:
        op = e.spec.nas_config.operations.operation.add()
        op.operation_type = op_type
        for pname, ptype, lst in specs:
            p = op.parameter_specs.parameters.add()
            p.name, p.parameter_type = pname, ptype
            p.feasible_space.list.extend(lst)
    return e


@pytest.fixture(scope="module")
def stub():
    server, port = serve(DispatchService([RandomService(), DartsService()]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch)
    ch.close()
    server.stop(0)


def _ask(s, exp, k):
    rep = s.GetSuggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=k))
    return [[(a.name, a.value) for a in pa.assignments] for pa in rep.parameter_assignments]


def _refused(s, exp, needle):
    with pytest.raises(grpc.RpcError) as ei:
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and needle in ei.value.details(), ei.value.details()
    with pytest.raises(grpc.RpcError) as ei:
        s.GetSuggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=1))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and needle in ei.value.details(), ei.value.details()


def test_katibs_example_experiment_gives_the_three_strings(stub):
    exp = make_experiment()
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    assert _ask(stub, exp, 1) == [[("algorithm-settings", DEFAULT_SETTINGS), ("search-space", SEARCH_SPACE), ("num-layers", "8")]]


def test_overriding_settings_keep_their_strings_in_the_default_order(stub):
    exp = make_experiment({"batch_size": "None", "num_epochs": 2, "w_lr": "0.01", "num_workers": 0})
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    want = ("{'num_epochs': '2', 'w_lr': '0.01', 'w_lr_min': 0.001, 'w_momentum': 0.9, 'w_weight_decay': 0.0003, "
            "'w_grad_clip': 5.0, 'alpha_lr': 0.0003, 'alpha_weight_decay': 0.001, 'batch_size': 'None', 'num_workers': '0', "
            "'init_channels': 16, 'print_step': 50, 'num_nodes': 4, 'stem_multiplier': 3}")
    assert _ask(stub, exp, 1) == [[("algorithm-settings", want), ("search-space", SEARCH_SPACE), ("num-layers", "8")]]


@pytest.mark.parametrize("k", [0, 1, 3])
def test_current_request_number_identical_lists(stub, k):
    exp = make_experiment(num_layers=3, operations=(("max_pooling", (("filter_size", api.CATEGORICAL, ("3", "7")),)),))
    got = _ask(stub, exp, k)
    assert got == [[("algorithm-settings", DEFAULT_SETTINGS), ("search-space", "['max_pooling_3x3', 'max_pooling_7x7']"),
                    ("num-layers", "3")]] * k


def test_only_the_first_spec_counts_and_skip_connection_ignores_its_specs(stub):
    ops = (("conv", (("filter_size", api.CATEGORICAL, ("1",)), ("other", api.INT, ()))),
           ("skip_connection", (("anything", api.INT, ()),)))
    assert _ask(stub, make_experiment(operations=ops), 1)[0][1] == ("search-space", "['conv_1x1', 'skip_connection']")


@pytest.mark.parametrize("name,value", [
    ("num_epochs", 0), ("num_epochs", "x"), ("num_epochs", "1.5"), ("num_epochs", "None"), ("batch_size", 0), ("batch_size", "none"),
    ("num_workers", -1), ("init_channels", 0), ("print_step", 0), ("num_nodes", 0), ("stem_multiplier", 0),
    ("w_lr", -0.1), ("w_lr", "nan"), ("w_lr", "None"), ("w_lr_min", -1), ("w_momentum", -1), ("w_weight_decay", "inf"),
    ("w_grad_clip", -1), ("alpha_lr", "x"), ("alpha_weight_decay", -1), ("bogus", 1)])
def test_bad_settings_are_refused_naming_the_setting(stub, name, value):
    _refused(stub, make_experiment({name: value}), name)


def test_good_settings_and_defaults():
    ok = {"num_epochs": "1", "w_lr": "0", "w_lr_min": "0", "w_momentum": "0.5", "w_weight_decay": "0", "w_grad_clip": "0",
          "alpha_lr": "1e-3", "alpha_weight_decay": "0", "batch_size": "None", "num_workers": "0", "init_channels": "1",
          "print_step": "1", "num_nodes": "1", "stem_multiplier": "1"}
    assert validate_darts_settings(ok) == ok and list(validate_darts_settings(ok)) == list(DEFAULTS)
    assert validate_darts_settings({}) == DEFAULTS


@pytest.mark.parametrize("kw,needle", [
    (dict(num_layers=0), "num_layers"), (dict(num_layers=-2), "num_layers"),
    (dict(operations=()), "at least one operation"),
    (dict(operations=(("", FILTERS),)), "operation_type"),
    (dict(operations=(("conv", ()),)), "'conv'"),
    (dict(operations=(("conv", (("filter_size", api.INT, ()),)),)), "CATEGORICAL"),
    (dict(operations=(("conv", (("filter_size", api.CATEGORICAL, ()),)),)), "non-empty"),
    (dict(algorithm="darts2"), "darts2"),
])
def test_nas_config_refusals(stub, kw, needle):
    _refused(stub, make_experiment(**kw), needle)
