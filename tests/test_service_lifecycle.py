"""Who owns a libkbo handle, and when it is closed: every engine through ``_lib.Handle`` (object first, then handle, once), and
every per-experiment cache of the services through ``_Base.experiment`` (one fingerprint per entry, bounded, closed on the way
out).  CPU only: the library is a recording stand-in and the CMA-ES sampler a host one."""
from __future__ import annotations

import pathlib

import numpy as np
import pytest
import torch

from kubeflow_b200 import _lib as L
from kubeflow_b200.suggestion import api_pb as api


# -- per-experiment cache of cmaes ------------------------------------------------------------------------------------------
class _T:
    def __init__(self, a): self.a = a
    def cpu(self): return self
    def numpy(self): return self.a


class _RecEs:
    """Stand-in for kubeflow_b200.cmaes.CmaEs: records its dimension, device and close."""
    made = []

    def __init__(self, mean0, sigma0, popsize=None, seed=0, device=0):
        self.D, self.popsize, self.device, self.closed = len(mean0), int(popsize or 8), device, 0
        self.r = np.random.default_rng(seed)
        _RecEs.made.append(self)

    def ask(self):
        return _T(self.r.uniform(0.05, 0.95, (self.popsize, self.D)))

    def close(self):
        self.closed += 1


@pytest.fixture
def rec(monkeypatch):
    import kubeflow_b200.cmaes as cm
    monkeypatch.setattr(cm, "CmaEs", _RecEs, raising=False)
    _RecEs.made = []
    return _RecEs


def _cma_experiment(name, n_params, settings=None):
    e = api.Experiment()
    e.name = name
    e.spec.objective.type = api.MINIMIZE
    e.spec.objective.objective_metric_name = "loss"
    e.spec.algorithm.algorithm_name = "cmaes"
    for k, v in (settings or {}).items():
        s = e.spec.algorithm.algorithm_settings.add()
        s.name, s.value = k, v
    for j in range(n_params):
        p = e.spec.parameter_specs.parameters.add()
        p.name, p.parameter_type = f"x{j}", api.DOUBLE
        p.feasible_space.min, p.feasible_space.max = "0", "1"
    return e


def _ask(svc, exp, k=3):
    return svc.get_suggestions(api.GetSuggestionsRequest(experiment=exp, current_request_number=k))


def test_cmaes_recreated_with_a_changed_space_gets_a_new_sampler(rec):
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    svc = CmaesService()
    _ask(svc, _cma_experiment("cma-re", 2))
    old = svc._exps["cma-re"].es
    rep = _ask(svc, _cma_experiment("cma-re", 3))               # deleted and recreated under the same name, one more parameter
    new = svc._exps["cma-re"].es
    assert new is not old and new.D == 3 and old.closed == 1 and new.closed == 0
    assert [len(pa.assignments) for pa in rep.parameter_assignments] == [3, 3, 3]
    _ask(svc, _cma_experiment("cma-re", 3))                      # unchanged: same sampler
    assert svc._exps["cma-re"].es is new


def test_cmaes_evicts_and_closes_the_least_recently_used_sampler(rec):
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    assert CmaesService().max_experiments == 64
    svc = CmaesService(max_experiments=2)
    for name in ("cma-a", "cma-b", "cma-a", "cma-c"):
        _ask(svc, _cma_experiment(name, 2))
    a, b, c = rec.made
    assert list(svc._exps) == ["cma-a", "cma-c"] and (a.closed, b.closed, c.closed) == (0, 1, 0)


def test_cmaes_samplers_go_to_the_service_device_unless_the_experiment_sets_one(rec):
    from kubeflow_b200.suggestion.cmaes_service import CmaesService
    svc = CmaesService({"device": 3})
    _ask(svc, _cma_experiment("cma-dev", 2))
    _ask(svc, _cma_experiment("cma-own", 2, {"device": "1"}))
    assert [es.device for es in rec.made] == [3, 1]


# -- one owner of the libkbo handle -----------------------------------------------------------------------------------------
class _FakeLib:
    """Records every kbo_* call; kbo_create and kbo_<kind>_create hand out non-null pointers, ``fail`` makes that create fail."""

    def __init__(self, fail=None):
        self.calls, self.fail = [], fail

    def __getattr__(self, name):
        if not name.startswith("kbo_"):
            raise AttributeError(name)

        def fn(*args):
            self.calls.append(name)
            if name == "kbo_last_error":
                return b"stand-in failure"
            if name == self.fail:
                return L.KBO_ERR_CUDA
            if name.endswith("_create"):
                args[0 if name == "kbo_create" else 1]._obj.value = 0x1000 + len(self.calls)
            return L.KBO_OK
        return fn


def _engines():
    from kubeflow_b200.cmaes import CmaEs
    from kubeflow_b200.enas import EnasController
    from kubeflow_b200.forest import ForestEngine
    from kubeflow_b200.gbrt import GbrtEngine
    from kubeflow_b200.gp import GPEngine
    from kubeflow_b200.mvtpe import MvTpe
    from kubeflow_b200.tpe import Tpe
    return {None: lambda: GPEngine(0),
            "tpe": lambda: Tpe([("uniform", 0.0, 1.0), ("choice", 3)]),
            "mvtpe": lambda: MvTpe([("float", 0.0, 1.0), ("cat", 3)]),
            "cma": lambda: CmaEs(np.zeros(2), 0.5, popsize=4),
            "forest": lambda: ForestEngine(0),
            "gbrt": lambda: GbrtEngine(0),
            "enas": lambda: EnasController(2, 8, 3)}


@pytest.fixture
def fake_cuda(monkeypatch):
    """A CUDA device as far as the engines' constructors can tell: the library records, device tensors live on the host."""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, device=None, **kw: empty(*a, **kw))

    def use(lib):
        monkeypatch.setattr(L, "load", lambda: lib)
        return lib
    return use


@pytest.mark.parametrize("kind", [None, "tpe", "mvtpe", "cma", "forest", "gbrt", "enas"])
def test_close_destroys_the_object_then_the_handle_once(fake_cuda, kind):
    lib = fake_cuda(_FakeLib())
    e = _engines()[kind]()
    assert isinstance(e, L.Handle)
    made = ["kbo_create"] + ([f"kbo_{kind}_create"] if kind else [])
    assert lib.calls == made
    e.close()
    assert lib.calls == made + ([f"kbo_{kind}_destroy"] if kind else []) + ["kbo_destroy"]
    n = len(lib.calls)
    e.close()
    del e
    assert len(lib.calls) == n


@pytest.mark.parametrize("kind", ["tpe", "mvtpe", "cma", "forest", "gbrt", "enas"])
def test_failed_object_create_destroys_the_handle_and_reports_its_error(fake_cuda, kind):
    lib = fake_cuda(_FakeLib(fail=f"kbo_{kind}_create"))
    try:
        _engines()[kind]()
    except L.KboError as err:      # the handle is gone by the time the error reaches the caller, not when it is collected
        assert "stand-in failure" in str(err)
        assert lib.calls == ["kbo_create", f"kbo_{kind}_create", "kbo_last_error", "kbo_destroy"]
    else:
        pytest.fail("no KboError")


@pytest.mark.parametrize("kind", ["tpe", "mvtpe", "cma", "forest", "gbrt", "enas"])    # GPEngine's text, now every engine's
def test_failed_kbo_create_has_one_message_and_nothing_to_destroy(fake_cuda, kind):
    lib = fake_cuda(_FakeLib(fail="kbo_create"))
    with pytest.raises(L.KboError, match=r"kbo_create failed \(no usable CUDA device\?\)"):
        _engines()[kind]()
    assert lib.calls == ["kbo_create"]


def test_optimizer_close_closes_its_engine():
    from kubeflow_b200.optimizer import Optimizer
    from kubeflow_b200.space import Real

    class Eng:
        closed = 0

        def close(self):
            Eng.closed += 1
    opt = Optimizer([Real(0.0, 1.0)], engine=Eng())
    opt.close()
    opt.close()
    assert Eng.closed == 1 and opt._engine is None


def test_only_the_handle_owner_creates_or_finalises_handles():
    root = pathlib.Path(L.__file__).parent
    hits = sorted({str(p.relative_to(root)) for p in root.rglob("*.py") for token in ("kbo_create(", "__del__")
                   if token in p.read_text()})
    assert hits == ["_lib.py"]
