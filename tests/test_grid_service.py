"""CPU: Katib's ``grid`` algorithm through a real in-process gRPC server — the hand-worked grid covered point by point, then
the fallback order; seeds; a restarted service; a recreated experiment; every refusal with its message; a grid of 10¹² points
drawn from without building it, and the grid-size limit."""
import itertools
import os
import tracemalloc

import grpc
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.grid_service import MAX_POINTS, MAX_VALUES, Grid, GridService
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService, RandomService
from tests.test_grpc_service import add_trial

RUNNING = api.TRIAL_CONDITIONS.index("RUNNING")

# Experiment order lr, layers, opt; sorted by name layers, lr, opt: 4 × 11 × 2 = 88 points
PARAMS = (("lr", api.DOUBLE, "0.0", "1.0", "0.1", ()), ("layers", api.INT, "1", "7", "2", ()),
          ("opt", api.CATEGORICAL, None, None, None, ("sgd", "adam")))
LR = ["0.0", "0.1", "0.2", "0.30000000000000004", "0.4", "0.5", "0.6000000000000001", "0.7000000000000001", "0.8", "0.9", "1.0"]
LAYERS = ["1", "3", "5", "7"]
OPT = ["sgd", "adam"]
ALL = {(lr, n, o) for lr in LR for n in LAYERS for o in OPT}


def make_experiment(params=PARAMS, settings=None, name="grid-1", max_trial_count=0, algorithm="grid"):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = algorithm
    e.spec.max_trial_count = max_trial_count
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for pname, ptype, lo, hi, step, lst in params:
        p = e.spec.parameter_specs.parameters.add()
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
    svc = GridService()
    server, port = serve(DispatchService([RandomService(), svc]), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    yield SuggestionStub(ch), svc
    ch.close()
    server.stop(0)


def _ask(s, req, k):
    req.current_request_number = k
    rep = s.GetSuggestions(req)
    assert len(rep.parameter_assignments) == k
    return [tuple((a.name, a.value) for a in pa.assignments) for pa in rep.parameter_assignments]


def _values(points):
    return [tuple(v for _, v in p) for p in points]


def _refused(s, exp, *needles):
    with pytest.raises(grpc.RpcError) as ei:
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=exp))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT, ei.value.details()
    for needle in needles:
        assert needle in ei.value.details(), ei.value.details()


def test_values_and_the_mixed_radix_order_of_the_names():
    exp = make_experiment()
    g = Grid(exp.spec.parameter_specs.parameters)
    assert g.size == 88 and [repr(v) for v in g.values[0]] == LR and g.values[1] == [1, 3, 5, 7] and g.values[2] == OPT
    assert g.point(0) == [0.0, 1, "sgd"] and g.point(1) == [0.0, 1, "adam"]     # opt, the last name, varies fastest
    assert g.point(2) == [0.1, 1, "sgd"] and g.point(22) == [0.0, 3, "sgd"]     # then lr, then layers
    for i in range(88):
        pa = api.GetSuggestionsReply().parameter_assignments.add()
        for name, v in zip(("lr", "layers", "opt"), g.point(i)):
            a = pa.assignments.add()
            a.name, a.value = name, repr(v) if name == "lr" else str(v)
        assert g.id_of(reversed(pa.assignments)) == i                            # matched by name, not position
    bad = api.GetSuggestionsReply().parameter_assignments.add()
    for name, v in (("lr", "0.3"), ("layers", "1"), ("opt", "sgd")):              # 0.3 is not arange's 0.30000000000000004
        a = bad.assignments.add()
        a.name, a.value = name, v
    assert g.id_of(bad.assignments) is None
    trim = make_experiment(params=(("x", api.DOUBLE, "0.0", "0.3", "0.1", ()),))
    assert Grid(trim.spec.parameter_specs.parameters).values == [[0.0, 0.1, 0.2]]   # arange's 0.30000000000000004 > 0.3 dropped
    no_step = make_experiment(params=(("n", api.INT, "2", "5", None, ()), ("d", api.DISCRETE, None, None, None, ("16", "32"))))
    assert Grid(no_step.spec.parameter_specs.parameters).values == [[2, 3, 4, 5], ["16", "32"]]


def test_full_coverage_then_the_fallback_order(stub):
    s, svc = stub
    req = api.GetSuggestionsRequest(experiment=make_experiment(settings={"random_state": 3}, name="grid-cover"))
    issued, held, n = [], [], 0
    conditions = (api.SUCCEEDED, RUNNING, api.FAILED)
    for k in (5, 13, 1, 30, 39):                  # 88 points over five calls
        pts = _ask(s, req, k)
        assert all([name for name, _ in p] == ["lr", "layers", "opt"] for p in pts)
        issued += _values(pts)
        for p in held + pts[:-1]:                # the last point of each call comes back one call later: in flight meanwhile
            add_trial(req, f"t{n}", dict(p), 0.5, condition=conditions[n % 3])
            n += 1
        held = pts[-1:]
    assert len(issued) == 88 and set(issued) == ALL
    # every point visited or in flight: only points not finished are drawn, the running trials and the one held back
    not_finished = {tuple(a.value for a in t.spec.parameter_assignments.assignments) for t in req.trials
                    if t.status.condition == RUNNING} | set(_values(held))
    assert len(not_finished) == 30
    again = _values(_ask(s, req, 40))
    assert set(again) <= not_finished and len(set(again)) > 1
    # every point finished: any point of the grid
    for p in held:
        add_trial(req, f"t{n}", dict(p), 0.5)
    for t in req.trials:
        t.status.condition = api.SUCCEEDED
    last = _values(_ask(s, req, 200))
    assert set(last) <= ALL and len(set(last)) > 30


def test_equal_seeds_give_equal_sequences_and_other_seeds_other_ones(stub):
    s, _ = stub

    def run(seed, name):
        req = api.GetSuggestionsRequest(experiment=make_experiment(settings={"random_state": seed}, name=name))
        out = []
        for k in (3, 4, 5):
            pts = _ask(s, req, k)
            out += _values(pts)
            for p in pts:
                add_trial(req, f"t{len(req.trials)}", dict(p), 0.1)
        return out

    a, b, c = run(11, "grid-seed-a"), run(11, "grid-seed-b"), run(12, "grid-seed-c")
    assert a == b and a != c and len(set(a)) == len(set(c)) == 12


def test_a_restarted_service_issues_only_the_points_katib_does_not_have():
    server, port = serve(GridService(), port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    s = SuggestionStub(ch)
    req = api.GetSuggestionsRequest(experiment=make_experiment(settings={"random_state": 5}, name="grid-restart"))
    ordered = sorted(ALL)
    have = ordered[::2]
    for i, p in enumerate(have):
        add_trial(req, f"old-{i}", dict(zip(("lr", "layers", "opt"), p)), 0.2,
                  condition=(api.SUCCEEDED, RUNNING, api.FAILED, api.KILLED)[i % 4])
    got = _values(_ask(s, req, 20)) + _values(_ask(s, req, 24))
    assert sorted(got) == ordered[1::2]
    ch.close()
    server.stop(0)


def test_a_recreated_experiment_starts_clean(stub):
    s, svc = stub
    one = (("x", api.INT, "1", "4", "1", ()),)
    req = api.GetSuggestionsRequest(experiment=make_experiment(params=one, settings={"random_state": 1}, name="grid-recreate"))
    first = _values(_ask(s, req, 3))
    old = svc._exps["grid-recreate"]
    assert len(set(first)) == 3 and len(old.issued) == 3
    two = (("x", api.INT, "1", "4", "1", ()), ("y", api.CATEGORICAL, None, None, None, ("a",)))
    req = api.GetSuggestionsRequest(experiment=make_experiment(params=two, settings={"random_state": 1}, name="grid-recreate"))
    second = _values(_ask(s, req, 4))
    new = svc._exps["grid-recreate"]
    assert new is not old and sorted(second) == [(str(x), "a") for x in range(1, 5)]     # the old in-flight ids are gone
    assert len(new.issued) == 4


@pytest.mark.parametrize("params,settings,max_trial_count,needles", [
    ((("lr", api.DOUBLE, "0", "1", None, ()),), {}, 0, ("'lr'", "step > 0")),
    ((("lr", api.DOUBLE, "0", "1", "0", ()),), {}, 0, ("'lr'", "step > 0")),
    ((("lr", api.DOUBLE, "0", "1", "-0.5", ()),), {}, 0, ("'lr'", "step > 0")),
    ((("n", api.INT, "1", "9", "0", ()),), {}, 0, ("'n'", "step > 0")),
    ((("n", api.INT, "1", "9", "-2", ()),), {}, 0, ("'n'", "step > 0")),
    ((("n", api.INT, "one", "9", "1", ()),), {}, 0, ("'n'", "must be numbers")),
    ((("n", api.INT, "1", "nine", "1", ()),), {}, 0, ("'n'", "must be numbers")),
    ((("n", api.INT, "1", "9", "two", ()),), {}, 0, ("'n'", "must be numbers")),
    ((("lr", api.DOUBLE, "0", "1", "tenth", ()),), {}, 0, ("'lr'", "must be numbers")),
    (PARAMS, {"bogus": 1}, 0, ("unknown setting bogus",)),
    (PARAMS, {"random_state": -1}, 0, ("random_state",)),
    (PARAMS, {"random_state": "x"}, 0, ("random_state",)),
    (PARAMS, {}, 89, ("89", "88")),
    ((("n", api.INT, "0", str(MAX_VALUES), "1", ()),), {}, 0, ("'n'", f"limit of {MAX_VALUES} values")),
    ((("x", api.INT, "1", "3", "1", ()), ("x", api.CATEGORICAL, None, None, None, ("a",))), {}, 0, ("unique", "'x'")),
])
def test_refusals_name_the_parameter_or_setting(stub, params, settings, max_trial_count, needles):
    _refused(stub[0], make_experiment(params=params, settings=settings, max_trial_count=max_trial_count), *needles)


def test_accepted_edges(stub):
    s = stub[0]
    for mtc in (0, 1, 88):
        s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(max_trial_count=mtc)))
    s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(settings={"random_state": 0})))
    _refused(s, make_experiment(algorithm="grid2"), "grid2")


def test_a_grid_of_a_trillion_points_is_drawn_from_without_building_it(stub):
    s, _ = stub
    big = tuple((c, api.INT, "1", "1000", "1", ()) for c in "abcd")            # 1000⁴ = 10¹² points
    req = api.GetSuggestionsRequest(experiment=make_experiment(params=big, settings={"random_state": 9}, name="grid-big"))
    _ask(s, req, 1)                                                             # warm: first-call allocations out of the count
    tracemalloc.start()
    try:
        seen = []
        for _ in range(3):
            pts = _values(_ask(s, req, 100))
            seen += pts
            for p in pts[:50]:
                add_trial(req, f"t{len(req.trials)}", dict(zip("abcd", p)), 1.0)
        _, peak = tracemalloc.get_traced_memory()
    finally:
        tracemalloc.stop()
    assert peak < 8 << 20, f"peak {peak} bytes"
    assert len(set(seen)) == 300 and all(1 <= int(v) <= 1000 for p in seen for v in p)


def test_the_grid_size_limit_is_refused_by_name(stub):
    s = stub[0]
    # 2¹⁶ · 2¹⁶ · 2¹⁶ · 2¹⁴ = 2⁶² points: exactly the limit
    at = tuple((c, api.INT, "1", str(1 << b), "1", ()) for c, b in zip("abcd", (16, 16, 16, 14)))
    assert Grid(make_experiment(params=at).spec.parameter_specs.parameters).size == MAX_POINTS == 1 << 62
    s.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=make_experiment(params=at)))
    over = at[:3] + (("d", api.INT, "0", str(1 << 14), "1", ()),)
    _refused(s, make_experiment(params=over), f"limit of {MAX_POINTS} points", str(MAX_POINTS + (1 << 48)))


def test_product_order_matches_itertools_over_sorted_names():
    params = (("zeta", api.CATEGORICAL, None, None, None, ("p", "q")), ("alpha", api.INT, "0", "2", "1", ()),
              ("mid", api.DISCRETE, None, None, None, ("8", "4")))
    g = Grid(make_experiment(params=params).spec.parameter_specs.parameters)
    ref = [dict(zip(("alpha", "mid", "zeta"), c)) for c in itertools.product([0, 1, 2], ["8", "4"], ["p", "q"])]
    assert [dict(zip(("zeta", "alpha", "mid"), g.point(i))) for i in range(g.size)] == ref


def test_the_example_experiment_is_a_valid_grid_of_48_points():
    yaml = pytest.importorskip("yaml")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "deploy", "experiment-grid-example.yaml")) as f:
        spec = yaml.safe_load(f)["spec"]
    types = {"double": api.DOUBLE, "int": api.INT, "categorical": api.CATEGORICAL, "discrete": api.DISCRETE}
    params = tuple((p["name"], types[p["parameterType"]], p["feasibleSpace"].get("min"), p["feasibleSpace"].get("max"),
                    p["feasibleSpace"].get("step"), p["feasibleSpace"].get("list", ())) for p in spec["parameters"])
    exp = make_experiment(params=params, settings={s["name"]: s["value"] for s in spec["algorithm"]["algorithmSettings"]},
                          max_trial_count=spec["maxTrialCount"], algorithm=spec["algorithm"]["algorithmName"])
    GridService().validate(exp)
    assert Grid(exp.spec.parameter_specs.parameters).size == spec["maxTrialCount"] == 48
