"""CPU: Katib's ``pbt`` algorithm over a real in-process gRPC server — settings validation, simulated Experiments of more
than ten generations whose trials carry a counter through their checkpoint directories, replayed call by call in the oracle
(oracle/pbt_oracle.py) on the same draws, a restart mid-run, batches larger than the free slots, hostile names, and routing."""
import json
import math
import os
import re

import grpc
import numpy as np
import pytest

from kubeflow_b200.suggestion import api_pb as api
from kubeflow_b200.suggestion.pbt_service import (GENERATION, PARENT, PREDECESSOR, PbtService, PbtTrial, call_rng, plan,
                                                  validate_pbt_settings)
from kubeflow_b200.suggestion.internal import HyperParameterSearchSpace
from kubeflow_b200.suggestion.server import SuggestionStub, serve
from kubeflow_b200.suggestion.service import DispatchService
from oracle import pbt_oracle as O

DNS_LABEL = re.compile(r"[a-z0-9]([-a-z0-9]{0,61}[a-z0-9])?")
SPACE = [("lr", api.DOUBLE, "0.01", "1.0", []), ("layers", api.INT, "1", "8", []),
         ("batch", api.DISCRETE, "", "", ["16", "32", "64", "128"]), ("opt", api.CATEGORICAL, "", "", ["sgd", "adam", "ftrl"])]
TYPES = {api.DOUBLE: "double", api.INT: "int", api.DISCRETE: "discrete", api.CATEGORICAL: "categorical"}
ORACLE_SPACE = [{"name": n, "type": TYPES[t], "min": lo, "max": hi, "list": lst} for n, t, lo, hi, lst in SPACE]
RUNNING = api.TRIAL_CONDITIONS.index("RUNNING")
CONDITIONS = {api.SUCCEEDED: "succeeded", api.EARLYSTOPPED: "succeeded", api.FAILED: "failed", api.KILLED: "failed",
              api.METRICSUNAVAILABLE: "failed"}


def pbt_experiment(settings, name="pbt-exp", objective=api.MAXIMIZE, space=SPACE):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = objective
    e.spec.objective.objective_metric_name = "score"
    e.spec.algorithm.algorithm_name = "pbt"
    for k, v in settings.items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, str(v)
    for n, t, lo, hi, lst in space:
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = n, t
        p.feasible_space.min, p.feasible_space.max = lo, hi
        p.feasible_space.list.extend(lst)
    return e


def serve_stub(service):
    server, port = serve(service, port=0, host="127.0.0.1")
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    return server, ch, SuggestionStub(ch)


@pytest.fixture(scope="module")
def stub():
    server, ch, s = serve_stub(DispatchService([PbtService()]))
    yield s
    ch.close()
    server.stop(0)


def replies(reply):
    return [(pa.trial_name, {a.name: a.value for a in pa.assignments}, dict(pa.labels)) for pa in reply.parameter_assignments]


def oracle_population(req, pending=()):
    out = []
    for t in req.trials:
        y = next((float(m.value) for m in t.status.observation.metrics if m.name == "score"), None)
        out.append(dict(name=t.name, generation=int(t.spec.labels.get(GENERATION, "0")), parent=t.spec.labels.get(PARENT),
                        predecessor=t.spec.labels.get(PREDECESSOR), params={a.name: a.value for a in t.spec.parameter_assignments.assignments},
                        objective=y, condition=CONDITIONS.get(t.status.condition, "running")))
    for name, params, labels in pending:
        out.append(dict(name=name, generation=int(labels[GENERATION]), parent=labels.get(PARENT), predecessor=labels.get(PREDECESSOR),
                        params=params, objective=None, condition="running"))
    return out


def oracle_step(req, k, pending=()):
    exp = req.experiment
    st = validate_pbt_settings({s.name: s.value for s in exp.spec.algorithm.algorithm_settings})
    pop = oracle_population(req, pending)
    rng = call_rng(st["random_state"], exp.name, [t["name"] for t in pop])
    goal = "MAXIMIZE" if exp.spec.objective.type == api.MAXIMIZE else "MINIMIZE"
    return [(o["trial_name"], o["params"], o["labels"]) for o in O.step(pop, ORACLE_SPACE, goal, st, rng, k, exp.name)]


def gain(p):
    """The toy problem: progress per trial, best at lr = 0.3, 6 layers, batch 64, adam."""
    return (1.0 - 2.0 * (float(p["lr"]) - 0.3) ** 2 - 0.02 * (int(p["layers"]) - 6) ** 2 - 0.1 * abs(math.log2(int(p["batch"]) / 64))
            + {"sgd": 0.0, "adam": 0.3, "ftrl": 0.1}[p["opt"]])


def add_trial(req, name, params, labels):
    t = req.trials.add()
    t.name = name
    t.spec.objective.objective_metric_name = "score"
    for k, v in params.items():
        a = t.spec.parameter_assignments.assignments.add()
        a.name, a.value = k, v
    t.spec.labels.update(labels)
    t.status.condition = RUNNING
    return t


def run_trial(root, t, outcome):
    """Reads the counter of the trial's checkpoint directory, adds its progress, writes it back and reports it."""
    path = os.path.join(root, t.name, "state.json")
    progress = json.load(open(path))["progress"] if os.path.exists(path) else 0.0
    progress += gain({a.name: a.value for a in t.spec.parameter_assignments.assignments})
    with open(path, "w") as f:
        json.dump({"progress": progress}, f)
    t.status.condition = api.FAILED if outcome == "failed" else api.SUCCEEDED
    if outcome == "ok":
        m = t.status.observation.metrics.add()
        m.name, m.value = "score", repr(progress)


def snapshot(d):
    return {n: open(os.path.join(d, n), "rb").read() for n in sorted(os.listdir(d))} if os.path.isdir(d) else None


class Sim:
    """A Katib-like driver: asks for trials up to its parallelism, runs the oldest half of the running ones each round."""

    def __init__(self, root, n_pop, seed=5, name="pbt-exp", objective=api.MAXIMIZE, parallel=None):
        self.root, self.n_pop = str(root), n_pop
        self.parallel = parallel or max(n_pop // 2, 1)
        self.req = api.GetSuggestionsRequest(experiment=pbt_experiment(
            {"suggestion_trial_dir": self.root, "n_population": n_pop, "truncation_threshold": 0.25, "resample_probability": 0.1,
             "random_state": seed}, name=name, objective=objective))
        self.running, self.names, self.done = [], set(), 0

    def ask(self, stub):
        k = self.parallel - len(self.running)
        told = {t.name for t in self.req.trials}
        files = {n: snapshot(os.path.join(self.root, n)) for n in told}
        expect = oracle_step(self.req, k)
        self.req.current_request_number = k
        got = replies(stub.GetSuggestions(self.req))
        assert got == expect                                                  # decision for decision, on the same draws
        for name, params, labels in got:
            assert DNS_LABEL.fullmatch(name) and len(name) <= 63 and name not in self.names
            self.names.add(name)
            parent, pred = labels.get(PARENT), labels.get(PREDECESSOR)
            assert pred is None or pred in told
            if parent is None:
                assert labels[GENERATION] == "0" and snapshot(os.path.join(self.root, name)) == {}
            else:
                assert parent in told
                assert int(labels[GENERATION]) == int(next(t for t in self.req.trials if t.name == parent).spec.labels[GENERATION]) + 1
                assert snapshot(os.path.join(self.root, name)) == files[parent]    # the parent's files at hand-off
            add_trial(self.req, name, params, labels)
            self.running.append(name)
        return got

    def run(self):
        by_name = {t.name: t for t in self.req.trials}
        for name in self.running[:max(len(self.running) // 2, 1)]:
            self.done += 1
            outcome = "failed" if self.done % 29 == 0 else "no metric" if self.done % 31 == 0 else "ok"
            run_trial(self.root, by_name[name], outcome)
        self.running = self.running[max(len(self.running) // 2, 1):]

    def current(self):
        superseded = {t.spec.labels.get(PREDECESSOR) for t in self.req.trials}
        return [t for t in self.req.trials if t.name not in superseded]

    def best(self):
        vals = [float(m.value) for t in self.req.trials for m in t.status.observation.metrics]
        return max(vals) if vals else None

    def max_generation(self):
        return max((int(t.spec.labels[GENERATION]) for t in self.req.trials), default=0)


def members_gain(sim):
    return float(np.mean([gain({a.name: a.value for a in t.spec.parameter_assignments.assignments}) for t in sim.current()]))


@pytest.mark.parametrize("n_pop", [8, 40])
def test_simulated_experiment_agrees_with_the_oracle(stub, tmp_path, n_pop):
    sim = Sim(tmp_path, n_pop)
    while sim.max_generation() < 10:
        sim.ask(stub)
        assert len(sim.current()) == min(len(sim.req.trials), n_pop)     # one current trial per slot
        sim.run()
    roots = sim.req.trials[:n_pop]                                        # generation 0 fills the population first
    assert all(PREDECESSOR not in t.spec.labels and PARENT not in t.spec.labels for t in roots)
    first_gain = float(np.mean([gain({a.name: a.value for a in t.spec.parameter_assignments.assignments}) for t in roots]))
    # the toy problem improves: the best objective grows and the population's hyperparameters move toward the optimum
    first = [float(m.value) for t in roots for m in t.status.observation.metrics]
    assert sim.best() > 5 * max(first)
    assert members_gain(sim) > first_gain
    assert any(t.status.condition == api.FAILED for t in sim.req.trials)
    fresh = [t for t in sim.req.trials if PREDECESSOR in t.spec.labels and PARENT not in t.spec.labels]
    assert fresh and all(t.spec.labels[GENERATION] == "0" for t in fresh)


def test_minimize_experiment_agrees_with_the_oracle(stub, tmp_path):
    sim = Sim(tmp_path, 6, seed=11, name="pbt-min", objective=api.MINIMIZE, parallel=6)
    while sim.max_generation() < 10:
        sim.ask(stub)
        sim.run()
    exploited = [t for t in sim.req.trials if t.spec.labels.get(PARENT) not in (None, t.spec.labels.get(PREDECESSOR))]
    assert exploited


def test_restart_gives_the_same_next_assignments(tmp_path):
    servers = [serve_stub(DispatchService([PbtService()])) for _ in range(2)]
    sim = Sim(tmp_path, 8, seed=3)
    while sim.max_generation() < 5:
        sim.ask(servers[0][2])
        sim.run()
    req = api.GetSuggestionsRequest()
    req.CopyFrom(sim.req)
    req.current_request_number = sim.parallel - len(sim.running)
    before = sim.ask(servers[0][2])
    assert before and replies(servers[1][2].GetSuggestions(req)) == before     # a fresh service: state lives in the trials
    while sim.max_generation() < 10:                                            # ... and it carries on
        sim.ask(servers[1][2])
        sim.run()
    for server, ch, _ in servers:
        ch.close()
        server.stop(0)


def test_batches_return_fewer_and_pending_names_are_not_reissued(stub, tmp_path):
    req = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(tmp_path), "n_population": 6,
                                                               "random_state": 1}, name="batch"), current_request_number=10)
    first = replies(stub.GetSuggestions(req))
    assert len(first) == 6 and len({n for n, _, _ in first}) == 6
    assert replies(stub.GetSuggestions(req)) == []                           # every slot has a trial pending
    for name, params, labels in first[:3]:
        add_trial(req, name, params, labels)
    assert replies(stub.GetSuggestions(req)) == []                           # three seen, three still pending
    for t in req.trials[:2]:
        run_trial(str(tmp_path), t, "ok")
    second = replies(stub.GetSuggestions(req))
    pending = first[3:]
    assert second == oracle_step(req, 10, pending)
    assert len(second) == 2 and {lab[PREDECESSOR] for _, _, lab in second} == {req.trials[0].name, req.trials[1].name}
    assert not {n for n, _, _ in second} & {n for n, _, _ in first}
    assert replies(stub.GetSuggestions(req)) == []                           # again before they come back: nothing new
    for name, params, labels in second + first[3:]:
        add_trial(req, name, params, labels)
    assert replies(stub.GetSuggestions(req)) == []                           # all back: every slot still busy


def test_zero_requested_returns_nothing(stub, tmp_path):
    req = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(tmp_path)}, name="zero"))
    assert replies(stub.GetSuggestions(req)) == [] and os.listdir(tmp_path) == []


def tree(d):
    return sorted(os.path.relpath(os.path.join(p, n), d) for p, ds, fs in os.walk(d) for n in ds + fs)


def test_hostile_names_write_nothing_outside_the_trial_dir(stub, tmp_path):
    root = tmp_path / "trials"
    root.mkdir()
    (tmp_path / "x").mkdir()
    (tmp_path / "x" / "secret").write_text("s")
    before = [p for p in tree(tmp_path) if not p.startswith("trials")]
    req = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(root), "n_population": 5},
                                                              name="../x"), current_request_number=5)
    got = replies(stub.GetSuggestions(req))
    assert len(got) == 5 and all(n.startswith("x-") and DNS_LABEL.fullmatch(n) for n, _, _ in got)
    assert sorted(os.listdir(root)) == sorted(n for n, _, _ in got)
    assert [p for p in tree(tmp_path) if not p.startswith("trials")] == before
    # a trial name that would resolve outside the directory is refused before anything is written
    for bad in ("../x", "..", "a/b", "A"):
        r = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(root), "n_population": 5}, name="h2"),
                                      current_request_number=5)
        t = add_trial(r, bad, {"lr": "0.5", "layers": "2", "batch": "16", "opt": "sgd"}, {GENERATION: "0"})
        t.status.condition = api.SUCCEEDED
        m = t.status.observation.metrics.add()
        m.name, m.value = "score", "1.0"
        with pytest.raises(grpc.RpcError) as ei:
            stub.GetSuggestions(r)
        assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and repr(bad) in ei.value.details()
    assert [p for p in tree(tmp_path) if not p.startswith("trials")] == before and len(os.listdir(root)) == 5


def test_parent_without_a_directory_gives_an_empty_one(stub, tmp_path):
    req = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(tmp_path), "n_population": 5,
                                                               "random_state": 2}, name="nodir"), current_request_number=5)
    for name, params, labels in replies(stub.GetSuggestions(req)):
        t = add_trial(req, name, params, labels)
        os.rmdir(tmp_path / name)                                            # the trial never wrote one
        t.status.condition = api.SUCCEEDED
        m = t.status.observation.metrics.add()
        m.name, m.value = "score", "1.0"
    got = replies(stub.GetSuggestions(req))
    assert len(got) == 5 and all(lab.get(PARENT) and os.listdir(tmp_path / n) == [] for n, _, lab in got)


def test_missing_trial_dir_is_refused(stub, tmp_path):
    req = api.GetSuggestionsRequest(experiment=pbt_experiment({"suggestion_trial_dir": str(tmp_path / "nope")}, name="nope"),
                                    current_request_number=1)
    with pytest.raises(grpc.RpcError) as ei:
        stub.GetSuggestions(req)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and "suggestion_trial_dir" in ei.value.details()


def test_plan_agrees_with_the_oracle_on_random_populations():
    """Populations the simulation rarely reaches: ties, overlapping ends (threshold > 0.5), failures everywhere, EARLYSTOPPED."""
    ss = HyperParameterSearchSpace.convert(pbt_experiment({}, objective=api.MINIMIZE))
    conds = ["running", "succeeded", "failed"]
    for case in range(200):
        g = np.random.default_rng(case)
        pop, names = [], []
        for i in range(int(g.integers(0, 30))):
            cond = conds[int(g.integers(0, 3))]
            obj = float(g.integers(0, 4)) if cond == "succeeded" and g.random() < 0.9 else None
            pred = names[int(g.integers(0, len(names)))] if names and g.random() < 0.5 else None
            parent = (pred if g.random() < 0.5 else names[int(g.integers(0, len(names)))]) if pred else None
            params = {"lr": repr(float(g.uniform(0.01, 1.0))), "layers": str(int(g.integers(1, 9))),
                      "batch": ["16", "32", "64", "128"][int(g.integers(0, 4))], "opt": ["sgd", "adam", "ftrl"][int(g.integers(0, 3))]}
            pop.append(dict(name=f"t{i}", generation=int(g.integers(0, 4)), parent=parent, predecessor=pred, params=params,
                            objective=obj, condition=cond))
            names.append(f"t{i}")
        pop = [t for t in pop if t["predecessor"] is None or sum(u["predecessor"] == t["predecessor"] for u in pop) == 1]
        st = {"n_population": int(g.integers(5, 12)), "truncation_threshold": float(g.choice([0.2, 0.5, 0.75, 0.9])),
              "resample_probability": [None, 0.0, 0.3, 1.0][case % 4]}
        state = {"running": "in flight", "succeeded": "completed", "failed": "ended"}
        trials = [PbtTrial(t["name"], t["generation"], t["parent"], t["predecessor"], t["params"], t["objective"],
                           "ended" if t["condition"] == "succeeded" and t["objective"] is None else state[t["condition"]]) for t in pop]
        k = int(g.integers(0, 15))
        got = [(t.name, t.values, t.labels()) for t in plan(trials, ss, st, np.random.default_rng([case, 1]), k, "exp")]
        want = [(o["trial_name"], o["params"], o["labels"]) for o in O.step(pop, ORACLE_SPACE, "MINIMIZE", st,
                                                                             np.random.default_rng([case, 1]), k, "exp")]
        assert got == want, case


# ---- validation -----------------------------------------------------------------------------------------------------------
def _validate(stub, settings, space=SPACE):
    stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=pbt_experiment(settings, space=space)))


@pytest.mark.parametrize("settings,frag", [
    ({}, "suggestion_trial_dir"), ({"suggestion_trial_dir": ""}, "suggestion_trial_dir"),
    ({"suggestion_trial_dir": "relative/dir"}, "suggestion_trial_dir"),
    ({"n_population": 4}, "n_population"), ({"n_population": "many"}, "n_population"), ({"n_population": "5.5"}, "n_population"),
    ({"truncation_threshold": 0}, "truncation_threshold"), ({"truncation_threshold": 1}, "truncation_threshold"),
    ({"truncation_threshold": "nan"}, "truncation_threshold"), ({"truncation_threshold": "x"}, "truncation_threshold"),
    ({"resample_probability": -0.1}, "resample_probability"), ({"resample_probability": 1.5}, "resample_probability"),
    ({"resample_probability": "often"}, "resample_probability"),
    ({"random_state": -1}, "random_state"), ({"random_state": "seed"}, "random_state"),
    ({"n_generations": 3}, "n_generations"),
])
def test_validation_names_the_setting(stub, settings, frag):
    full = {"suggestion_trial_dir": "/ckpt", **settings}
    if settings == {}:
        full = {}
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, full)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and frag in ei.value.details()


def test_validation_accepts_the_settings_and_every_parameter_type(stub):
    _validate(stub, {"suggestion_trial_dir": "/ckpt"})
    _validate(stub, {"suggestion_trial_dir": "/ckpt", "n_population": 5, "truncation_threshold": 0.5, "resample_probability": 0,
                     "random_state": 0})
    _validate(stub, {"suggestion_trial_dir": "/ckpt", "n_population": 400, "truncation_threshold": 0.01, "resample_probability": 1})
    for spec in SPACE:
        _validate(stub, {"suggestion_trial_dir": "/ckpt"}, space=[spec])
    assert validate_pbt_settings({"suggestion_trial_dir": "/c"}) == {"suggestion_trial_dir": "/c", "n_population": 40,
                                                                    "truncation_threshold": 0.2, "resample_probability": None}


@pytest.mark.parametrize("space,frag", [([("lr", api.DOUBLE, "1.0", "0.5", [])], "min < max"), ([("opt", api.CATEGORICAL, "", "", [])], "empty"),
                                        ([("x", api.UNKNOWN_TYPE, "0", "1", [])], "parameter_type"), ([], "no parameters")])
def test_validation_refuses_bad_spaces(stub, space, frag):
    with pytest.raises(grpc.RpcError) as ei:
        _validate(stub, {"suggestion_trial_dir": "/ckpt"}, space=space)
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and frag in ei.value.details()


# ---- dispatch -------------------------------------------------------------------------------------------------------------
def test_dispatch_routes_pbt_and_every_other_algorithm():
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    from kubeflow_b200.suggestion.enas_service import EnasService
    from kubeflow_b200.suggestion.hyperband import HyperbandService
    from kubeflow_b200.suggestion.mvtpe_service import MultivariateTpeService
    from kubeflow_b200.suggestion.service import RandomService, SkoptService, SobolService
    from kubeflow_b200.suggestion.tpe_service import TpeService
    services = [SkoptService(), RandomService(), SobolService(), CmaesService(), TpeService(), MultivariateTpeService(), EnasService(),
                HyperbandService(), PbtService()]
    d = DispatchService(services)
    for svc in services:
        for name in svc.algorithm_names:
            e = pbt_experiment({})
            e.spec.algorithm.algorithm_name = name
            assert d._pick(e) is svc
    assert sorted(d._by_name) == ["bayesianoptimization", "cmaes", "enas", "hyperband", "multivariate-tpe", "pbt", "random", "sobol",
                                  "tpe"]
    server, ch, stub = serve_stub(d)
    _validate(stub, {"suggestion_trial_dir": "/ckpt"})
    e = pbt_experiment({})
    e.spec.algorithm.algorithm_name = "grid"
    with pytest.raises(grpc.RpcError) as ei:
        stub.ValidateAlgorithmSettings(api.ValidateAlgorithmSettingsRequest(experiment=e))
    assert ei.value.code() == grpc.StatusCode.INVALID_ARGUMENT and "'pbt'" in ei.value.details() and "'grid'" in ei.value.details()
    ch.close()
    server.stop(0)
