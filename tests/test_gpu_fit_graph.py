"""The fit's factorisation replayed as one cached CUDA graph against the same schedule enqueued call by call
(kbo_debug_fit_stream_path): L, W, alpha, the LML and info must agree bit for bit, since the graph holds the same kernels,
arguments and dependencies.  Covered: partitioned (N = 8192) and unpartitioned (N = 1000, 1800) fits, Matérn and RBF, lazy and
full inverse; a second fit with new y and θ that replays the graph; a new N that rebuilds it; buffers moved by a larger
reservation (the executable graph is updated in place); append and rebase after a graph fit; a non-positive-definite K; two
handles on one device; and where the graph's kernel nodes run when the chain has its own SM partition."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gp_oracle as O             # noqa: E402
from kubeflow_b200 import _lib as Lb          # noqa: E402
from kubeflow_b200.gp import GPEngine         # noqa: E402
from tests import _fit_scale as H             # noqa: E402

pytestmark = pytest.mark.gpu


def stats(e):
    s = (C.c_int32 * 8)()
    Lb.check(e.lib, e._h, e.lib.kbo_debug_fit_graph(e._h, s))
    return dict(captures=s[0], updates=s[1], instantiations=s[2], replays=s[3], chain=s[4], rest=s[5], other=s[6], launches=s[7])


def engine(kind, mode, stream_path, D):
    th = O.theta_of_record(D)
    e = GPEngine(0, kernel=kind, acq="ei", var_mode=mode, length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    if stream_path:
        Lb.check(e.lib, e._h, e.lib.kbo_debug_fit_stream_path(e._h, 1))
    return e


def bits(t):
    return t.contiguous().view(torch.int64)


def snapshot(e):
    """info, LML, L and alpha as the fit left them (a lazy fit's missing rows of W are not formed), then all of W."""
    rc, info = H.fit_info(e)
    lml = e.fit_info()["lml"] if rc == 0 else None
    Lm, _, al = H.state(e, with_w=False)
    out = dict(rc=rc, info=info, lml=lml, L=bits(Lm), alpha=bits(al))
    if rc == 0:
        out["W"] = bits(H.state(e)[1])
    return out


def assert_same(g, r, where):
    a, b = snapshot(g), snapshot(r)
    assert (a["rc"], a["info"]) == (b["rc"], b["info"]), f"{where}: status {a['rc'], a['info']} vs {b['rc'], b['info']}"
    assert a["lml"] == b["lml"], f"{where}: LML {a['lml']!r} vs {b['lml']!r}"
    for k in ("L", "alpha", "W"):
        if k in a:
            assert torch.equal(a[k], b[k]), f"{where}: {k} differs in {int((a[k] != b[k]).sum())} entries"
    return a


def set_theta(e, amplitude, ls_scale, noise):
    e.amplitude, e.noise = amplitude, noise
    e.length_scale = e.length_scale * ls_scale


# N = 1000 is below the size a lazy inverse pays at (its leading rows would be all of W): N = 1800 is the unpartitioned lazy case
CASES = [(8192, "matern52", "tc"), (8192, "rbf", "f64"), (8192, "rbf", "tc"), (1000, "matern52", "f64"), (1000, "rbf", "tc"),
         (1800, "matern52", "tc"), (1800, "rbf", "f64")]


@pytest.mark.parametrize("N,kind,mode", CASES)
def test_graph_fit_is_the_stream_fit_bit_for_bit_and_follows_new_data(N, kind, mode):
    D = 32 if N == 8192 else 8
    X, y, Xc = O.synthetic(N, 4096, D)
    g, r = engine(kind, mode, False, D), engine(kind, mode, True, D)
    for e in (g, r):
        e.tell(X, y)
        e.ask(Xc)   # the sweep sets what the next fit's lazy inverse keeps
    s0 = stats(g)
    assert s0["captures"] >= 1 and stats(r)["captures"] == 0
    for e in (g, r):
        e.tell(X, y)
    first = assert_same(g, r, f"N={N} {kind} {mode}")
    s1 = stats(g)
    assert s1["captures"] == s0["captures"] and s1["replays"] == s0["replays"] + 1, (s0, s1)
    # new y and θ on the same handle: the graph is replayed, and alpha must follow the new data (θ reaches the Gram node)
    y2 = 2.0 * y[::-1].copy() + 0.3
    for e in (g, r):
        set_theta(e, 1.7, 0.8, 2e-3)
        e.tell(X, y2)
    second = assert_same(g, r, f"N={N} {kind} {mode}, new y and θ")
    s2 = stats(g)
    assert s2["captures"] == s1["captures"] and s2["replays"] == s1["replays"] + 1, (s1, s2)
    assert not torch.equal(first["alpha"], second["alpha"]) and not torch.equal(first["L"], second["L"])
    bg, br = g.ask(Xc), r.ask(Xc)
    assert (bg.index, bg.value, bg.mu, bg.std) == (br.index, br.value, br.mu, br.std)
    g.close()
    r.close()


def test_graph_is_rebuilt_for_a_new_size_and_updated_when_buffers_move():
    D = 8
    g, r = engine("matern52", "f64", False, D), engine("matern52", "f64", True, D)
    for N in (1800, 3000, 1800):
        X, y, _ = O.synthetic(N, 1, D)
        before = stats(g)
        for e in (g, r):
            e.tell(X, y)
        assert_same(g, r, f"N={N}")
        after = stats(g)
        assert after["captures"] == before["captures"] + 1 and after["instantiations"] == before["instantiations"] + 1, (before, after)
    # a larger kbo_trtri on the handle reallocates its scratch plane: the same N then captures the same topology over a moved
    # buffer, and the executable graph is updated in place
    n2 = 4096
    Lt = torch.eye(n2, dtype=torch.float64, device="cuda")
    Wt = torch.empty(n2, n2, dtype=torch.float64, device="cuda")
    Lb.check(g.lib, g._h, g.lib.kbo_trtri(g._h, Lt.data_ptr(), n2, n2, Wt.data_ptr(), n2, g._stream()))
    torch.cuda.synchronize()
    X, y, _ = O.synthetic(1800, 1, D)
    y = y + 0.25
    before = stats(g)
    for e in (g, r):
        e.tell(X, y)
    assert_same(g, r, "N=1800 after the scratch plane moved")
    after = stats(g)
    assert after["captures"] == before["captures"] + 1 and after["updates"] == before["updates"] + 1, (before, after)
    assert after["instantiations"] == before["instantiations"], (before, after)
    g.close()
    r.close()


@pytest.mark.parametrize("N,mode", [(8150, "tc"), (1000, "f64")])
def test_append_and_rebase_after_a_graph_fit(N, mode):
    D = 32 if N > 4096 else 8
    X, y, Xc = O.synthetic(N + 3, 2048, D)
    g, r = engine("matern52", mode, False, D), engine("matern52", mode, True, D)
    for e in (g, r):
        e.tell(X[:N], y[:N])
        e.ask(Xc)
        e.tell(X[:N], y[:N])
        for i in range(N, N + 3):
            e.append(X[i], float(y[i]))
    assert stats(g)["replays"] >= 2
    assert_same(g, r, f"N={N}: three appends")
    for e in (g, r):
        e.rebase(N - 10, y[:N - 10] * 0.5)
    assert_same(g, r, f"N={N}: rebase")
    g.close()
    r.close()


@pytest.mark.parametrize("N,p", [(4096, 2985), (1000, 257)])
def test_a_non_positive_definite_K_reports_the_same_pivot(N, p):
    X, y = O.not_pd_at(N, p)
    g, r = H.pivot_engine("f64"), H.pivot_engine("f64")
    Lb.check(r.lib, r._h, r.lib.kbo_debug_fit_stream_path(r._h, 1))
    f = (p - 1) // 64 * 64   # the rows factored before the failing 64-block
    for rep in range(2):   # captured, then replayed
        for e in (g, r):
            try:
                e.tell(X, y)
            except Lb.KboError:
                pass
        # past the failing block L is not defined: which kernels still ran there after the pivot was flagged depends on how the
        # streams interleaved, in either path
        (rg, ig), (rr, ir) = H.fit_info(g), H.fit_info(r)
        assert (rg, ig) == (rr, ir) and ig == p, ((rg, ig), (rr, ir))
        Lg, Lr = H.state(g, with_w=False)[0], H.state(r, with_w=False)[0]
        assert torch.equal(bits(Lg[:f, :f]), bits(Lr[:f, :f])), f"N={N} p={p} fit {rep}: the factored rows differ"
    assert stats(g)["replays"] == 2
    # a good history on the same handle replays the graph and recovers
    Xg, yg, _ = O.synthetic(N, 1, 4)
    for e in (g, r):
        e.noise = 1e-3
        e.tell(Xg, yg)
    assert assert_same(g, r, f"N={N} good fit after a failed one")["info"] == 0
    g.close()
    r.close()


def test_two_handles_on_one_device_keep_their_own_graphs():
    D = 16
    (Xa, ya, _), (Xb, yb, _) = O.synthetic(4096, 1, D), O.synthetic(3000, 1, D)
    yb = yb * 3.0 - 1.0
    ga, gb, r = engine("matern52", "f64", False, D), engine("matern52", "f64", False, D), engine("matern52", "f64", True, D)
    for rep in range(2):
        ga.tell(Xa, ya)
        gb.tell(Xb, yb)
        r.tell(Xa, ya)
        assert_same(ga, r, f"handle a, fit {rep}")
        r.tell(Xb, yb)
        assert_same(gb, r, f"handle b, fit {rep}")
    for e in (ga, gb):
        s = stats(e)
        assert s["captures"] == 1 and s["replays"] == 2, s
    for e in (ga, gb, r):
        e.close()


def test_graph_kernel_nodes_run_in_the_partition_their_stream_belongs_to():
    """At N = 8192 the chain, its near shadows and W_PP run on the chain's 8 SMs: per panel four factorisations, three solves and
    three updates, six W_PP products, and (all panels but the last) four solves, three updates and the next diagonal block's
    update — 32·16 + 31·8 = 760 kernel nodes in the chain's green context.  The Gram launch runs on the caller's side; everything
    else in the rest's green context."""
    D = 32
    X, y, _ = O.synthetic(8192, 1, D)
    g = engine("matern52", "f64", False, D)
    g.tell(X, y)
    torch.cuda.synchronize()
    s = stats(g)
    print("graph:", s)
    if s["chain"] == 0 and s["rest"] == 0:
        pytest.skip("this device or driver gives the fit no SM partition (green contexts)")
    assert s["chain"] == 32 * 16 + 31 * 8, s
    assert s["other"] == 1, s
    assert s["chain"] + s["rest"] + s["other"] == s["launches"], s
    g.close()
