"""GPU parity tests: the CUDA path (through the C ABI in include/kbo.h) against the CPU oracle and the
golden vectors produced by the real scikit-learn GPR.  Tolerances: FP64 mode 1e-8 on mu/std/acq; tensor-core
mode 1e-5 on the acquisition value (BASELINE.json north_star), argmax index equal unless the oracle's own
top-2 gap is below the tolerance (then the GPU pick must be within tolerance of the oracle maximum)."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

TOL_TC = 1e-5
TOL_F64 = 1e-8


def _engine(g_or_kw, var_mode, **over):
    from kubeflow_b200.gp import GPEngine
    kw = dict(kernel=g_or_kw["kind"], length_scale=g_or_kw["length_scale"], amplitude=g_or_kw["amplitude"],
              noise=g_or_kw["noise"], acq=g_or_kw.get("acq_kind", g_or_kw.get("acq", "ei")), xi=g_or_kw["xi"],
              kappa=g_or_kw["kappa"], var_mode=var_mode)
    kw.update(over)
    return GPEngine(0, **kw)


def _same(a, b, tol=1e-10):
    """Same suggestion: identical index, value / mu / std equal to FP64 rounding.  (Bit-equality held while every path ended in the
    same W-based FP64 evaluation; a lazy fit evaluates the survivors by panel solves with L, an eager one through W = L⁻¹.)"""
    return (a.index == b.index and abs(a.value - b.value) <= tol * max(1.0, abs(b.value)) and abs(a.mu - b.mu) <= tol * max(1.0, abs(b.mu))
            and abs(a.std - b.std) <= 1e-8 * max(1.0, abs(b.std)))


def _check_argmax(best, acq_ref, tol):
    i_ref = int(np.argmax(acq_ref))
    if best.index != i_ref:
        assert abs(acq_ref[best.index] - acq_ref[i_ref]) <= tol, (best.index, i_ref, acq_ref[best.index], acq_ref[i_ref])
    assert abs(best.value - acq_ref[i_ref]) <= tol


@pytest.mark.parametrize("var_mode,tol", [("f64", TOL_F64), ("auto", TOL_F64), ("tc", TOL_TC)])
def test_golden(golden, var_mode, tol):
    """f64 / auto (the default: FP64 for problems this small) must match to 1e-8.  Forced tensor-core mode is held to the
    1e-5 contract for EI and PI; for LCB the value is -(mu - kappa*sigma), so the error is kappa*d(sigma) with
    d(sigma) = d(var)/(2 sigma): the fp16x3 contraction's d(var) ~ 1e-6 is amplified at sigma ~ 1e-2 (tiny, ill-conditioned
    low-D histories) — there the bound is 5e-5 and `auto` never sends such problems to the tensor cores (DESIGN.md)."""
    if var_mode == "tc" and golden["acq_kind"] == "lcb":
        tol = 5e-5
    eng = _engine(golden, var_mode)
    eng.tell(golden["X"], golden["y"])
    info = eng.fit_info()
    assert info["info"] == 0
    assert abs(info["y_mean"] - golden["y_mean"]) < 1e-12 and abs(info["y_std"] - golden["y_std"]) < 1e-12
    assert abs(info["lml"] - golden["lml"]) < 1e-7 * max(1.0, abs(golden["lml"]))
    best, mu, std, acq = eng.ask(golden["Xc"], return_arrays=True)
    mu, std, acq = mu.cpu().numpy(), std.cpu().numpy(), acq.cpu().numpy()
    mtol = tol if var_mode != "tc" else 2e-6   # TC mode carries mu in fp32
    np.testing.assert_allclose(mu, golden["mu"], rtol=0, atol=mtol)
    np.testing.assert_allclose(std, golden["std"], rtol=0, atol=max(tol, 1e-7) if var_mode != "tc" else 5e-5)
    np.testing.assert_allclose(acq, golden["acq"], rtol=0, atol=tol)
    _check_argmax(best, golden["acq"], tol)
    assert abs(best.mu - golden["mu"][best.index]) < 1e-5 and abs(best.std - golden["std"][best.index]) < 1e-4
    # the array-free call is the product path (fp32 fast acquisition in tc mode): same winner, same value within tol
    b2 = eng.ask(golden["Xc"])
    _check_argmax(b2, golden["acq"], max(tol, 1e-6) if var_mode == "tc" else tol)
    eng.close()


def test_fit_state_blocks(golden):
    eng = _engine(golden, "f64")
    eng.tell(golden["X"], golden["y"])
    L, W, alpha = (t.cpu().numpy() for t in eng.state())
    np.testing.assert_allclose(L, golden["L"], rtol=0, atol=1e-11)
    np.testing.assert_allclose(W @ golden["L"], np.eye(len(golden["y"])), atol=1e-9)
    np.testing.assert_allclose(alpha, golden["alpha"], rtol=1e-8, atol=1e-9)
    eng.close()


@pytest.mark.parametrize("N,D,kind", [(1, 1, "rbf"), (63, 2, "matern52"), (64, 3, "rbf"), (65, 3, "matern52"), (130, 5, "rbf"),
                                      (257, 7, "matern52"), (700, 16, "matern52"), (1000, 8, "rbf")])
def test_building_blocks_gram_potrf_trtri(N, D, kind):
    """kbo_gram / kbo_potrf / kbo_trtri one at a time on caller-owned memory, ragged sizes around the 64-block."""
    import ctypes as C
    from kubeflow_b200 import _lib as Lb
    lib = Lb.load()
    h = C.c_void_p()
    assert lib.kbo_create(C.byref(h), 0) == 0
    X, _, _ = O.synthetic(N, 1, D)
    ls = 0.3 * np.sqrt(D)
    Xs = torch.tensor(X / ls, device="cuda")
    ld = (N + 63) // 64 * 64
    K = torch.full((N, ld), float("nan"), dtype=torch.float64, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.kbo_gram(h, Xs.data_ptr(), N, D, Lb.KERNELS[kind], 1.3, 1e-3, K.data_ptr(), ld, st) == 0
    Kref = O.kernel_matrix(X, X, ls, kind, 1.3) + 1e-3 * np.eye(N)
    np.testing.assert_allclose(K[:, :N].cpu().numpy(), Kref, rtol=0, atol=1e-13)
    info = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.kbo_potrf(h, K.data_ptr(), N, ld, info.data_ptr(), st) == 0
    assert int(info.item()) == 0
    Lg = torch.tril(K[:, :N]).cpu().numpy()
    Lref = np.linalg.cholesky(Kref)
    np.testing.assert_allclose(Lg, Lref, rtol=0, atol=1e-11)
    W = torch.full((N, ld), float("nan"), dtype=torch.float64, device="cuda")
    assert lib.kbo_trtri(h, K.data_ptr(), N, ld, W.data_ptr(), ld, st) == 0
    Wg = W[:, :N].cpu().numpy()
    assert np.all(np.triu(Wg, 1) == 0)
    np.testing.assert_allclose(Wg @ Lref, np.eye(N), atol=1e-8)
    lib.kbo_destroy(h)


@pytest.mark.parametrize("N,M,D,kind,acq", [(1024, 4096, 8, "rbf", "ei"), (1024, 3000, 8, "matern52", "lcb"),
                                            (2048, 2048, 32, "matern52", "ei"), (777, 1234, 5, "rbf", "pi")])
@pytest.mark.parametrize("var_mode,tol", [("f64", TOL_F64), ("tc", TOL_TC)])
def test_oracle_midsize(N, M, D, kind, acq, var_mode, tol):
    """cfg2 / cfg3-shaped histories at sizes the oracle finishes in seconds (θ of record, SURVEY.md §8(d))."""
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    ref = O.suggest(X, y, Xc, kind=kind, acq=acq, **th)
    eng = _engine(dict(kind=kind, acq=acq, **th), var_mode)
    eng.tell(X, y)
    best, mu, std, a = eng.ask(Xc, return_arrays=True)
    a = a.cpu().numpy()
    err = np.abs(a - ref["acq"]).max()
    print(f"\n[{var_mode}] N={N} M={M} D={D} {kind}/{acq}: max|d acq|={err:.3e} max|d mu|={np.abs(mu.cpu().numpy()-ref['mu']).max():.3e} "
          f"max|d std|={np.abs(std.cpu().numpy()-ref['std']).max():.3e}")
    atol = tol if var_mode == "tc" else 2e-7   # f64 mode: limited by cond(K)·eps of either side, not by the GPU
    if var_mode == "tc" and acq == "lcb":
        atol = 5e-5   # forced tensor-core mode on a small low-D history: kappa*d(sigma) with sigma ~ 1e-2 (see test_golden)
    np.testing.assert_allclose(a, ref["acq"], rtol=0, atol=atol)
    _check_argmax(best, ref["acq"], atol)
    eng.close()


def test_cfg3_full_size_history_candidate_subsample():
    """BASELINE cfg3 at its full trial count (N=8192, D=32, Matern-5/2, EI), tensor-core mode, on a 4096-candidate slice of
    the 1M grid (the oracle needs ~1 s per 2048 candidates at this N): acquisition within 1e-5, same argmax."""
    N, M, D = 8192, 4096, 32
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    ref = O.suggest(X, y, Xc, kind="matern52", acq="ei", **th)
    eng = _engine(dict(kind="matern52", acq="ei", **th), "tc")
    eng.tell(X, y)
    best, mu, std, a = eng.ask(Xc.astype(np.float32).astype(np.float64), return_arrays=True)
    err = np.abs(a.cpu().numpy() - ref["acq"]).max()
    print(f"\n[tc] cfg3 N={N} D={D} M={M}: max|d acq|={err:.3e} max|d mu|={np.abs(mu.cpu().numpy()-ref['mu']).max():.3e} "
          f"max|d std|={np.abs(std.cpu().numpy()-ref['std']).max():.3e}  lml gpu={eng.fit_info()['lml']:.6f} oracle={ref['fit']['lml']:.6f}")
    assert err <= TOL_TC
    _check_argmax(best, ref["acq"], TOL_TC)
    assert abs(eng.fit_info()["lml"] - ref["fit"]["lml"]) < 1e-6 * abs(ref["fit"]["lml"])
    eng.close()


@pytest.mark.parametrize("k_span", [32, 256, 1024, 1 << 20])
@pytest.mark.parametrize("rows,Npad", [(128, 256), (256, 1024), (384, 2048), (128, 768)])
def test_tc_variance_kernel_raw(rows, Npad, k_span):
    """The wgmma kernel alone: fp16 hi/lo planes in, Σ_j (Σ_{k<=j} A[m,k]·B[j,k])² out, vs fp64 NumPy on the same planes."""
    import ctypes as C
    from kubeflow_b200 import _lib as Lb
    lib = Lb.load()
    h = C.c_void_p()
    assert lib.kbo_create(C.byref(h), 0) == 0
    r = np.random.default_rng(rows * 7 + Npad)
    A = r.random((rows, Npad)) * 0.9 + 0.05
    B = np.tril(r.standard_normal((Npad, Npad)) * 40.0)
    Ah = A.astype(np.float16); Al = (A - Ah.astype(np.float64)).astype(np.float16)
    Bh = B.astype(np.float16); Bl = (B - Bh.astype(np.float64)).astype(np.float16)
    A2, B2 = Ah.astype(np.float64), Bh.astype(np.float64)
    V = A2 @ B2.T + A2 @ Bl.astype(np.float64).T + Al.astype(np.float64) @ B2.T      # exactly the three products issued
    ref = (V * V).sum(1)
    t = lambda a: torch.tensor(a, device="cuda").contiguous()
    dAh, dAl, dBh, dBl = t(Ah), t(Al), t(Bh), t(Bl)
    scale = torch.tensor([1.0, 1.0], dtype=torch.float64, device="cuda")
    var = torch.empty(rows, dtype=torch.float32, device="cuda")
    ssq = torch.empty(rows, dtype=torch.float64, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.kbo_tc_variance_raw(h, dAh.data_ptr(), dAl.data_ptr(), rows, dBh.data_ptr(), dBl.data_ptr(), Npad, scale.data_ptr(),
                                 0.0, var.data_ptr(), ssq.data_ptr(), k_span, st)
    assert rc == 0, lib.kbo_last_error(h)
    torch.cuda.synchronize()
    got = ssq.cpu().numpy()
    rel = np.abs(got - ref) / ref
    print(f"\nrows={rows} Npad={Npad} k_span={k_span}: max rel err Σv² = {rel.max():.3e}, mean signed = {((got-ref)/ref).mean():+.3e}")
    assert rel.max() < 2e-5
    lib.kbo_destroy(h)


@pytest.mark.parametrize("var_mode,tol", [("f64", 2e-7), ("tc", TOL_TC)])
def test_multi_chunk_sweep_matches_oracle(var_mode, tol):
    """Force the candidate grid through several scratch chunks with a ragged tail (64 MiB scratch: 16 384-row chunks in tc
    mode at Npad = 1024 — 32 768 for the ranking pass, which keeps one plane —, 8 192-row chunks in f64 mode) and compare every
    candidate with the oracle."""
    N, M, D = 1000, 40_003, 6
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    ref = O.suggest(X, y, Xc, kind="matern52", acq="ei", **th)
    eng = _engine(dict(kind="matern52", acq="ei", **th), var_mode, scratch_limit=64 << 20)
    eng.tell(X, y)
    best, mu, std, a = eng.ask(Xc, return_arrays=True)
    err = np.abs(a.cpu().numpy() - ref["acq"]).max()
    print(f"\n[{var_mode}] multi-chunk N={N} M={M}: max|d acq|={err:.3e}")
    assert err <= tol
    _check_argmax(best, ref["acq"], tol)
    b_host, t = eng.suggest_host(X, y, Xc)
    assert t["chunks"] >= 2 and b_host.index == eng.ask(Xc).index
    eng.close()


@pytest.mark.parametrize("D", [1, 17, 64, 130])
def test_dimension_sweep(D):
    """D below, across and above the 32-dimension slab of the K* kernel (and D > 128: two+ slabs with a ragged last one)."""
    N, M = 150, 600
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    ls = np.linspace(0.7, 1.4, D) * th["length_scale"]          # anisotropic
    kw = dict(th, length_scale=ls)
    ref = O.suggest(X, y, Xc, kind="rbf", acq="ei", **kw)
    for var_mode, tol in (("f64", 1e-8), ("tc", TOL_TC)):
        eng = _engine(dict(kind="rbf", acq="ei", **kw), var_mode)
        eng.tell(X, y)
        best, mu, std, a = eng.ask(Xc, return_arrays=True)
        np.testing.assert_allclose(a.cpu().numpy(), ref["acq"], rtol=0, atol=tol)
        _check_argmax(best, ref["acq"], tol)
        eng.close()


@pytest.mark.parametrize("seed", range(16))
def test_fuzz_ragged_shapes(seed):
    """Seeded random shapes around every tile boundary of the path (64-row Cholesky blocks, 128×64 K* tiles, 256-column
    j-tiles, 4-candidate acquisition groups), random kernel / acquisition / ARD, fp32 or fp64 candidates, both modes."""
    r = np.random.default_rng(1000 + seed)
    N = int(r.choice([1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 511, 513]))
    M = int(r.choice([1, 2, 3, 4, 5, 127, 128, 129, 1000, 2049]))
    D = int(r.choice([1, 2, 3, 7, 16, 31, 32, 33, 40]))
    kind = str(r.choice(["rbf", "matern52"]))
    acq = str(r.choice(["ei", "pi", "lcb"]))
    X, y, Xc = O.synthetic(N, M, D)
    ls = (0.3 * np.sqrt(D)) * (r.uniform(0.7, 1.5, D) if r.random() < 0.5 else 1.0)
    kw = dict(length_scale=ls, amplitude=float(r.uniform(0.5, 2.0)), noise=1e-3, xi=0.01, kappa=1.96)
    if r.random() < 0.5:
        Xc = Xc.astype(np.float32)
    ref = O.suggest(X, y, np.asarray(Xc, dtype=np.float64), kind=kind, acq=acq, **kw)
    for var_mode, tol in (("f64", 1e-7), ("tc", 5e-5 if acq == "lcb" else TOL_TC)):
        eng = _engine(dict(kind=kind, acq=acq, **kw), var_mode)
        eng.tell(X, y)
        best, mu, std, a = eng.ask(Xc, return_arrays=True)
        err = np.abs(a.cpu().numpy() - ref["acq"]).max()
        assert err <= tol, (seed, N, M, D, kind, acq, var_mode, err)
        _check_argmax(best, ref["acq"], tol)
        _check_argmax(eng.ask(Xc), ref["acq"], max(tol, 1e-6))
        eng.close()


def test_lml_gradient_matches_sklearn_golden_and_oracle():
    """kbo_lml_grad vs the real scikit-learn `log_marginal_likelihood(eval_gradient=True)` (tests/golden/lmlgrad_cases.npz)
    and vs the oracle at a size that spans several 64×64 pair tiles, isotropic and ARD."""
    import os
    from kubeflow_b200.gp import GPEngine
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "lmlgrad_cases.npz"), allow_pickle=False)
    for n in sorted({k.split("__")[0] for k in z.files}):
        ls = z[f"{n}__ls"]
        eng = GPEngine(0, kernel=str(z[f"{n}__kind"]), length_scale=ls, amplitude=float(z[f"{n}__amp"]), noise=float(z[f"{n}__noise"]), var_mode="f64")
        eng.tell(z[f"{n}__X"], z[f"{n}__y"])
        lml, g = eng.lml_grad()
        assert abs(lml - float(z[f"{n}__lml"])) < 1e-9
        np.testing.assert_allclose(g, z[f"{n}__grad"], rtol=0, atol=1e-8)
        eng.close()
    for kind, ard in (("matern52", True), ("rbf", False)):
        X, y, _ = O.synthetic(333, 1, 7)
        ls = 0.3 * np.sqrt(7) * (np.linspace(0.8, 1.3, 7) if ard else 1.0)
        ref_lml, ref_g = O.lml_and_grad(X, y, kind=kind, length_scale=ls, amplitude=1.4, noise=2e-3)
        eng = GPEngine(0, kernel=kind, length_scale=ls, amplitude=1.4, noise=2e-3, var_mode="f64")
        eng.tell(X, y)
        lml, g = eng.lml_grad()
        assert abs(lml - ref_lml) < 1e-8 * abs(ref_lml)
        np.testing.assert_allclose(g, ref_g, rtol=1e-8, atol=1e-7)
        eng.close()


def test_tc_mode_suggestion_is_refined_in_fp64(golden):
    """Tensor-core mode re-evaluates every candidate within 2e-4 of its fp32 maximum on the FP64 path: the returned suggestion
    must then equal the FP64 mode's — same index as the oracle's first-index argmax, value / mu / std to FP64 accuracy — even
    where the arrays of the tensor-core sweep are only 1e-5 accurate."""
    e64 = _engine(golden, "f64"); e64.tell(golden["X"], golden["y"])
    b64 = e64.ask(golden["Xc"])
    etc = _engine(golden, "tc"); etc.tell(golden["X"], golden["y"])
    btc = etc.ask(golden["Xc"])
    n = etc.last_contenders()
    assert 1 <= n <= 4096
    i_ref = int(np.argmax(golden["acq"]))
    assert btc.index == b64.index == i_ref
    assert abs(btc.value - b64.value) <= 1e-10 * max(1.0, abs(b64.value)) and abs(btc.value - golden["acq"][i_ref]) <= TOL_F64
    assert abs(btc.mu - b64.mu) <= 1e-10 * max(1.0, abs(b64.mu)) and abs(btc.std - b64.std) <= 1e-10
    for e in (e64, etc):
        e.close()


def test_tc_refinement_resolves_near_ties_like_the_oracle():
    """Candidates that differ by less than the tensor-core error: copies of the winner nudged by 1e-9 in one coordinate have
    acquisition values ~1e-9 apart, far below what the fp16x3 variance resolves.  The refined pick must be the oracle's."""
    X, y, Xc = O.synthetic(512, 20000, 6)
    th = O.theta_of_record(6)
    ref = O.suggest(X, y, Xc, kind="matern52", acq="ei", **th)
    rng = np.random.default_rng(7)
    near = Xc[ref["index"]][None, :] + 1e-9 * rng.standard_normal((64, 6))
    Xn = np.concatenate([Xc[:9000], near[:32], Xc[9000:], near[32:]])
    refn = O.suggest(X, y, Xn, kind="matern52", acq="ei", **th)
    eng = _engine(dict(kind="matern52", acq="ei", **th), "tc"); eng.tell(X, y)
    b = eng.ask(Xn)
    assert eng.last_contenders() >= 65
    assert b.index == refn["index"] and abs(b.value - refn["value"]) <= TOL_F64
    # sharded over 4 ranks: every shard refines its own contenders, the (value, lowest index) maximum is the same point
    q = len(Xn) // 4
    parts = [eng.ask(Xn[s:s + q + 3], global_offset=s) for s in range(0, len(Xn), q + 3)]
    win = max(parts, key=lambda p: (p.value, -p.index))
    assert (win.index, win.value) == (b.index, b.value)
    eng.close()


def test_ties_duplicates_and_sharding():
    X, y, Xc = O.synthetic(96, 1000, 4)
    th = O.theta_of_record(4)
    for var_mode in ("f64", "tc"):
        eng = _engine(dict(kind="matern52", acq="ei", **th), var_mode)
        eng.tell(X, y)
        b0 = eng.ask(Xc)
        # duplicate the winner later AND earlier: identical rows give bit-identical values -> lowest index wins
        Xd = np.concatenate([Xc, Xc[b0.index:b0.index + 1]])
        assert eng.ask(Xd).index == b0.index
        j = 5 if b0.index != 5 else 6
        Xe = Xc.copy(); Xe[j] = Xc[b0.index]
        assert eng.ask(Xe).index == min(j, b0.index)
        # sharding the grid over R ranks: max over (value, lowest global index) == single sweep (SURVEY.md §8(e))
        parts = [eng.ask(Xc[s:s + 250], global_offset=s) for s in range(0, 1000, 250)]
        win = max(parts, key=lambda b: (b.value, -b.index))
        assert win.index == b0.index and win.value == b0.value
        # idempotence / determinism: bit-identical on repeat
        b1 = eng.ask(Xc)
        assert (b1.index, b1.value, b1.mu, b1.std) == (b0.index, b0.value, b0.mu, b0.std)
        eng.close()


def test_device_tensor_inputs_and_f32_candidates():
    X, y, Xc = O.synthetic(200, 777, 6)
    th = O.theta_of_record(6)
    eng = _engine(dict(kind="rbf", acq="ei", **th), "f64")
    eng.tell(X, y)
    b_host, _, _, a_host = eng.ask(Xc, return_arrays=True)
    eng.tell(torch.tensor(X, device="cuda"), torch.tensor(y, device="cuda"))
    b_dev, _, _, a_dev = eng.ask(torch.tensor(Xc, device="cuda"), return_arrays=True)
    assert torch.equal(a_host, a_dev) and b_host == b_dev
    Xc32 = Xc.astype(np.float32)
    ref = O.suggest(X, y, Xc32.astype(np.float64), kind="rbf", acq="ei", **th)
    b32, _, _, a32 = eng.ask(Xc32, return_arrays=True)
    np.testing.assert_allclose(a32.cpu().numpy(), ref["acq"], atol=2e-7)
    eng.close()


def test_edge_cases_and_errors():
    from kubeflow_b200 import _lib as Lb
    th = O.theta_of_record(2)
    eng = _engine(dict(kind="rbf", acq="ei", **th), "tc")
    X, y, Xc = O.synthetic(10, 7, 2)
    # M = 1 and M not a multiple of 4
    eng.tell(X, y)
    for M in (1, 3, 5, 7):
        ref = O.suggest(X, y, Xc[:M], kind="rbf", acq="ei", **th)
        b = eng.ask(Xc[:M])
        assert b.index == ref["index"] and abs(b.value - ref["value"]) < TOL_TC
    # candidate == training point: variance collapses, EI ~ 0 there, no NaN
    b, mu, std, a = eng.ask(np.concatenate([X[:3], Xc]), return_arrays=True)
    assert torch.isfinite(a).all() and (std >= 0).all()
    # duplicate trial rows with zero noise -> not positive definite, reported like sklearn's LinAlgError
    eng2 = _engine(dict(kind="rbf", acq="ei", **{**th, "noise": 0.0}), "f64")
    Xdup = np.concatenate([X, X[:1]]); ydup = np.concatenate([y, y[:1]])
    eng2.tell(Xdup, ydup)
    with pytest.raises(Lb.KboNotPositiveDefinite):
        eng2.fit_info()
    with pytest.raises(Lb.KboNotPositiveDefinite):
        eng2.ask(Xc)
    # invalid arguments
    with pytest.raises(Lb.KboInvalidArgument):
        _engine(dict(kind="rbf", acq="ei", **{**th, "length_scale": -1.0}), "f64").tell(X, y)
    with pytest.raises(Lb.KboInvalidArgument):
        _engine(dict(kind="rbf", acq="ei", **{**th, "length_scale": [1.0, 2.0, 3.0]}), "f64").tell(X, y)
    with pytest.raises(ValueError):
        eng.ask(np.zeros((4, 3)))
    from kubeflow_b200.gp import GPEngine
    with pytest.raises(Lb.KboError):
        GPEngine(0).ask(Xc)   # sweep before fit
    eng.close(); eng2.close()


def test_acq_argmax_f32_standalone():
    """The HBM-bound pass alone (8 B/candidate in, 4 B out) vs NumPy, incl. NaN handling and a late duplicate max."""
    from kubeflow_b200.gp import GPEngine
    r = np.random.default_rng(3)
    M = 1_000_003
    mu_n = r.standard_normal(M).astype(np.float32)
    var_n = (r.random(M) * 0.5).astype(np.float32)
    var_n[17] = -1e-3            # clamps to 0 -> EI 0
    for acq in ("ei", "lcb", "pi"):
        eng = GPEngine(0, acq=acq)
        mu = 0.7 * mu_n.astype(np.float64) + 0.2
        sd = np.sqrt(np.maximum(var_n.astype(np.float64), 0) * 0.49)
        ref = O.acquisition(mu, sd, -1.1, acq, 0.01, 1.96)
        out = torch.empty(M, dtype=torch.float32, device="cuda")
        b = eng.acq_argmax_f32(torch.tensor(mu_n, device="cuda"), torch.tensor(var_n, device="cuda"), y_mean=0.2, y_std=0.7,
                               y_opt=-1.1, acq_out=out, global_offset=10)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-5, atol=2e-6)
        i = int(np.argmax(ref))
        assert b.index - 10 == i or abs(ref[b.index - 10] - ref[i]) < 2e-6
        eng.close()


def test_suggest_host_end_to_end():
    X, y, Xc = O.synthetic(512, 5000, 8)
    th = O.theta_of_record(8)
    ref = O.suggest(X, y, Xc, kind="matern52", acq="ei", **th)
    eng = _engine(dict(kind="matern52", acq="ei", **th), "tc")
    best, t = eng.suggest_host(X, y, Xc)
    assert abs(best.value - ref["value"]) < TOL_TC
    assert best.index == ref["index"] or abs(ref["acq"][best.index] - ref["value"]) < TOL_TC
    assert t["launches"] > 0 and t["total_ms"] > 0 and t["var_kernel_ms"] > 0
    eng.close()


@pytest.mark.parametrize("N0,k,var_mode,kind", [(200, 5, "f64", "matern52"), (70, 3, "f64", "rbf"), (1100, 3, "tc", "matern52"), (1, 4, "f64", "rbf")])
def test_fit_append_matches_refit_and_oracle(N0, k, var_mode, kind):
    """kbo_fit_append (bordered Cholesky row + row of W) against a refit of the extended history and against the oracle:
    factors, alpha, y statistics, LML and the suggestion must agree as if the history had been told in one go."""
    D = 6
    X, y, Xc = O.synthetic(N0 + k, 5000, D)
    th = O.theta_of_record(D)
    kw = dict(kind=kind, acq="ei", **th)
    inc = _engine(kw, var_mode); inc.tell(X[:N0], y[:N0])
    assert inc.room() == (-N0) % 64
    for i in range(N0, N0 + k):
        inc.append(X[i], y[i])
    ref = _engine(kw, var_mode); ref.tell(X, y)
    for a, b in zip(inc.state(), ref.state()):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=0, atol=2e-10)
    ii, ir = inc.fit_info(), ref.fit_info()
    for key in ("y_mean", "y_std", "y_opt"):
        assert abs(ii[key] - ir[key]) <= 1e-13 * max(1.0, abs(ir[key]))
    assert abs(ii["lml"] - ir["lml"]) <= 1e-9 * max(1.0, abs(ir["lml"]))
    bi, mi, si, ai = inc.ask(Xc, return_arrays=True)
    br, mr, sr, ar = ref.ask(Xc, return_arrays=True)
    tol = 1e-9 if var_mode == "f64" else 2e-6
    np.testing.assert_allclose(ai.cpu().numpy(), ar.cpu().numpy(), rtol=0, atol=tol)
    np.testing.assert_allclose(mi.cpu().numpy(), mr.cpu().numpy(), rtol=0, atol=1e-9)
    assert bi.index == br.index and abs(bi.value - br.value) <= 1e-9
    orc = O.suggest(X, y, Xc, kind=kind, acq="ei", **th)
    _check_argmax(bi, orc["acq"], TOL_F64)            # f64 natively, tc through the FP64 refinement of the contenders
    gl, gg = inc.lml_grad()
    rl, rg = ref.lml_grad()
    np.testing.assert_allclose(gg, rg, rtol=1e-8, atol=1e-8)
    inc.close(); ref.close()


def test_fit_append_room_and_errors():
    from kubeflow_b200 import _lib as Lb
    X, y, _ = O.synthetic(64, 10, 3)
    eng = _engine(dict(kind="rbf", acq="ei", **O.theta_of_record(3)), "f64")
    with pytest.raises(Lb.KboError):
        eng.append(X[0], 0.0)                   # before tell
    eng.tell(X, y)
    assert eng.room() == 0
    with pytest.raises(Lb.KboError):
        eng.append(X[0] + 0.5, 0.0)             # the 64-row pitch is full: the caller refits
    eng.tell(X[:63], y[:63])
    with pytest.raises(ValueError):
        eng.append(X[63][:2], 0.0)
    eng.append(X[63], y[63])
    assert eng.room() == 0 and eng.N == 64
    eng.close()


def test_fit_rebase_drops_rows_and_replaces_targets():
    """kbo_fit_rebase keeps the leading rows of the factorisation (no refit) and takes new targets: state and suggestion must
    equal a fresh fit of the shorter history with those targets; rows can then be appended again."""
    D = 5
    X, y, Xc = O.synthetic(150, 3000, D)
    th = O.theta_of_record(D)
    kw = dict(kind="matern52", acq="ei", **th)
    eng = _engine(kw, "f64"); eng.tell(X[:140], y[:140])
    y2 = y.copy(); y2[100:] = y2[100:] * 0.5 - 0.2
    eng.rebase(130, y2[:130])
    assert eng.N == 130 and eng.room() == 192 - 130
    for i in range(130, 150):
        eng.append(X[i], y2[i])
    ref = _engine(kw, "f64"); ref.tell(X, y2)
    for a_, b_ in zip(eng.state(), ref.state()):
        np.testing.assert_allclose(a_.cpu().numpy(), b_.cpu().numpy(), rtol=0, atol=2e-10)
    be, _, _, ae = eng.ask(Xc, return_arrays=True)
    br, _, _, ar = ref.ask(Xc, return_arrays=True)
    np.testing.assert_allclose(ae.cpu().numpy(), ar.cpu().numpy(), rtol=0, atol=1e-9)
    assert be.index == br.index
    _check_argmax(be, O.suggest(X, y2, Xc, kind="matern52", acq="ei", **th)["acq"], TOL_F64)
    from kubeflow_b200 import _lib as Lb
    with pytest.raises(Lb.KboInvalidArgument):
        eng.rebase(0)
    with pytest.raises(Lb.KboInvalidArgument):
        eng.rebase(151)
    eng.close(); ref.close()


def test_optimizer_constant_liar_appends_instead_of_refitting():
    """ask(n_points=3) tells two constant lies: with `incremental` they are appended (kbo_fit_append), without it refitted as
    skopt does — the three suggested points must be the same.  The next request (history + one finished trial) drops the
    lies, keeps the common prefix and appends; a lie that became an observation at the same x only swaps the target; an
    edited early row falls back to a refit."""
    from kubeflow_b200.optimizer import Optimizer
    from kubeflow_b200.space import Real
    dims = [Real(0.0, 1.0, name=f"x{i}") for i in range(4)]
    rng = np.random.default_rng(3)
    X0 = rng.random((40, 4)).tolist()
    y0 = [float(np.sin(3 * sum(r))) for r in X0]
    outs, fits, later = [], [], []
    for inc in (True, False):
        opt = Optimizer(dims, n_initial_points=5, random_state=11, n_points=20000, incremental=inc)
        opt.tell(X0, y0)
        pts = opt.ask(n_points=3)
        outs.append(np.asarray(pts))
        fits.append(opt.last_fit)
        opt.tell([pts[0]], [0.123])          # engine: history + lie(pts0) + lie(pts1); new history: history + pts0 observed
        a1 = opt.ask(); f1 = opt.last_fit
        opt.tell([pts[2]], [0.456])          # a new row after the common prefix
        a2 = opt.ask(); f2 = opt.last_fit
        opt.ask(); f3 = opt.last_fit
        later.append(np.asarray([a1, a2]))
        if inc:
            assert (f1, f2, f3) == ("rebase", "append", "reuse")
            opt.Xi[3] = [0.5] * 4; opt._Xt[3] = opt.space.transform([opt.Xi[3]])[0]
            opt.ask()
            assert opt.last_fit == "fit"
        else:
            assert (f1, f2, f3) == ("fit", "fit", "fit")
    assert fits == ["append", "fit"]
    np.testing.assert_allclose(outs[0], outs[1], rtol=0, atol=0)
    np.testing.assert_allclose(later[0], later[1], rtol=0, atol=0)


@pytest.mark.parametrize("N,M,D,kind,acq", [(1024, 50000, 8, "rbf", "ei"), (2048, 30000, 32, "matern52", "ei"), (1500, 20000, 6, "matern52", "lcb"),
                                            (1200, 20000, 5, "rbf", "pi")])
def test_one_product_ranking_pass_returns_the_same_suggestion(N, M, D, kind, acq):
    """kbo_set_tc_fast: the array-free tensor-core sweep ranks with one fp16 product and lets the FP64 refinement decide among
    the candidates that could still be the maximum.  The returned suggestion must be the three-product sweep's, bit for bit
    (both end in the same FP64 evaluation), and the FP64 engine's to rounding; the ranking error it calibrates is reported."""
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    kw = dict(kind=kind, acq=acq, **th)
    fast = _engine(kw, "tc"); fast.tell(X, y)
    slow = _engine(kw, "tc", tc_fast=False); slow.tell(X, y)
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    bf, bs, b6 = fast.ask(Xc), slow.ask(Xc), e64.ask(Xc)
    assert _same(bf, bs)
    assert bf.index == b6.index and abs(bf.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value))
    assert 1 <= fast.last_contenders() <= 4096
    assert 1e-7 < fast.last_rank_error() < 0.5           # fp16 hi planes only: |d sigma²| ~ 1e-4 … 1e-3, 3e-2 on ill-conditioned low-D fits
    assert slow.last_rank_error() == 0.0
    # sharded over 3 ranks: each shard calibrates and prunes on its own rows, the exchange picks the same point
    parts = [fast.ask(Xc[s:s + 7000], global_offset=s) for s in range(0, M, 7000)]
    win = max(parts, key=lambda b: (b.value, -b.index))
    assert (win.index, win.value) == (bf.index, bf.value)
    for e in (fast, slow, e64):
        e.close()


def test_one_product_ranking_pass_falls_back_when_too_many_survive():
    """6000 identical candidates all survive the pruning (> 4096): the sweep is redone with three products and the pick is
    the lowest index, as the reference's argmin over identical values."""
    X, y, Xc = O.synthetic(300, 10, 4)
    th = O.theta_of_record(4)
    eng = _engine(dict(kind="matern52", acq="ei", **th), "tc"); eng.tell(X, y)
    b = eng.ask(np.repeat(Xc[:1], 6000, axis=0))
    assert b.index == 0 and eng.last_contenders() > 4096
    ref = O.suggest(X, y, Xc[:1], kind="matern52", acq="ei", **th)
    assert abs(b.value - ref["value"]) <= TOL_TC
    eng.close()


def test_rebase_then_append_across_a_256_boundary_in_tc_mode():
    """fit 300 -> rebase 250 (the fp16 planes shrink to 256) -> append past 256: the planes and the K* scratch must grow back
    with the history (a stale 256-wide extent dropped rows/columns of W and wrote past the K* scratch).  Compared against a
    refit of the same 262-trial history, per-candidate arrays and the suggestion."""
    D = 6
    X, y, Xc = O.synthetic(262, 4000, D)
    th = O.theta_of_record(D)
    kw = dict(kind="matern52", acq="ei", **th)
    eng = _engine(kw, "tc"); eng.tell(np.concatenate([X[:250], X[:50] * 0.5 + 0.25]), np.concatenate([y[:250], y[:50]]))
    eng.rebase(250, y[:250])
    for i in range(250, 262):
        eng.append(X[i], y[i])
    assert eng.N == 262
    ref = _engine(kw, "tc"); ref.tell(X, y)
    be, me, se, ae = eng.ask(Xc, return_arrays=True)
    br, mr, sr, ar = ref.ask(Xc, return_arrays=True)
    np.testing.assert_allclose(ae.cpu().numpy(), ar.cpu().numpy(), rtol=0, atol=2e-6)
    np.testing.assert_allclose(se.cpu().numpy(), sr.cpu().numpy(), rtol=0, atol=2e-5)
    assert be.index == br.index and abs(be.value - br.value) <= 1e-9
    b2, r2 = eng.ask(Xc), ref.ask(Xc)          # the array-free path (ranking pass + FP64 decision)
    assert b2.index == r2.index and abs(b2.value - r2.value) <= 1e-9
    _check_argmax(b2, O.suggest(X, y, Xc, kind="matern52", acq="ei", **th)["acq"], TOL_F64)
    eng.close(); ref.close()


# ---- round 2: tensor-core K* generation + wgmma ranking kernel --------------------------------------------------------
@pytest.mark.parametrize("N,M,D,kind", [(1000, 700, 7, "matern52"), (2048, 1500, 32, "matern52"), (777, 300, 5, "rbf"), (1300, 513, 100, "matern52"),
                                        (300, 256, 40, "rbf")])
def test_tensor_core_kstar_plane_and_mean_against_fp64_kernel(N, M, D, kind):
    """tc_kstar.cu: K̃* from wgmma dot products + fp32 kernel evaluation vs the FP64 K* kernel of the same fit.  The fp16 hi
    planes may differ by one fp16 ulp where the fp32 value falls on the other side of a rounding boundary, nowhere by more;
    padding columns are zero; the on-the-fly mean agrees to the fp32 evaluation error times |alpha|."""
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    eng = _engine(dict(kind=kind, acq="ei", **th), "tc"); eng.tell(X, y)
    xc = torch.tensor(Xc.astype(np.float32), device="cuda")
    mu0, v0, p0 = eng.rank_pass(xc, 0, want_plane=True)
    mu1, v1, p1 = eng.rank_pass(xc, 1, want_plane=True)
    p0, p1 = p0.float().cpu().numpy(), p1.float().cpu().numpy()
    assert np.all(p1[:, N:] == 0) and np.all(p0[:, N:] == 0)
    Kref = O.kernel_matrix(Xc.astype(np.float32).astype(np.float64), X, th["length_scale"], kind, th["amplitude"])
    ulp = np.maximum(np.abs(Kref), 2.0 ** -14) * 2.0 ** -10       # one fp16 ulp at the value's magnitude (normal range)
    d = np.abs(p1[:, :N] - p0[:, :N])
    assert np.all(d <= 1.01 * ulp), f"max plane difference {np.max(d / ulp):.2f} ulp"
    frac = float(np.mean(d > 0))
    assert frac < 0.02, f"{frac:.4f} of the entries round differently"
    assert np.all(np.abs(p1[:, :N] - Kref) <= 0.51 * ulp + 2e-6)
    fit = O.gp_fit(X, y, kind=kind, **{k: th[k] for k in ("length_scale", "amplitude", "noise")})
    a1 = float(np.abs(fit["alpha"]).sum())
    dm = np.abs(mu1.cpu().numpy() - mu0.cpu().numpy()).max()
    print(f"\nN={N} M={M} D={D} {kind}: plane entries differing {frac:.2e}, max|d mu_n|={dm:.3e} (|alpha|_1={a1:.3e}), "
          f"max|d var_n|={np.abs(v1.cpu().numpy() - v0.cpu().numpy()).max():.3e}")
    assert dm <= 2e-6 * a1 + 1e-6
    # both ranking passes against the oracle's normalised posterior: the hi-plane-only contraction is a RANKING value
    mu_ref, std_ref = O.gp_predict(fit, Xc.astype(np.float32).astype(np.float64))
    var_ref = (std_ref / fit["y_std"]) ** 2
    for v in (v0, v1):
        assert np.abs(v.cpu().numpy() - var_ref).max() < 5e-2
    assert np.abs(v1.cpu().numpy() - v0.cpu().numpy()).max() < 1e-2
    np.testing.assert_allclose(mu1.cpu().numpy(), (mu_ref - fit["y_mean"]) / fit["y_std"], rtol=0, atol=2e-6 * a1 + 1e-5)
    eng.close()


@pytest.mark.parametrize("N,M,D,kind,acq", [(1024, 50000, 8, "rbf", "ei"), (2048, 30000, 32, "matern52", "ei"), (1500, 20000, 6, "matern52", "lcb"),
                                            (1200, 20000, 5, "rbf", "pi"), (1100, 9000, 70, "matern52", "ei")])
def test_tensor_core_ranking_pass_returns_the_fp64_suggestion(N, M, D, kind, acq):
    """The product path (prefix-bound pruning pass, tensor-core K*, wgmma ranking kernel, stratified calibration with a
    mean bound, FP64 decision) returns the same suggestion as the same path without the pruning pass, the round-1 ranking pass
    (FP64 K*), the three-product sweep and the FP64 engine."""
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    kw = dict(kind=kind, acq=acq, **th)
    new = _engine(kw, "tc"); new.tell(X, y)
    full = _engine(kw, "tc", rank_prefix=0); full.tell(X, y)
    old = _engine(kw, "tc", rank_tc=False); old.tell(X, y)
    slow = _engine(kw, "tc", tc_fast=False); slow.tell(X, y)
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    bn, bf, bo, bs, b6 = new.ask(Xc), full.ask(Xc), old.ask(Xc), slow.ask(Xc), e64.ask(Xc)
    assert _same(bn, bf)
    assert full.last_prefix_survivors() == -1 and new.last_prefix_survivors() >= 1
    full.close()
    assert _same(bn, bo) and _same(bn, bs) and (bo.index, bo.value, bo.mu, bo.std) == (bs.index, bs.value, bs.mu, bs.std)
    assert bn.index == b6.index and abs(bn.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value))
    assert new.last_unrefined() == 0 and 1 <= new.last_contenders() <= 4096
    # the round-1 ranking pass takes its mean from the FP64 K* kernel, as the calibration rows do: they differ only by the summation
    # order of the trial-tile split the kernel uses when it has few rows
    assert 0 < new.last_rank_mu_error() < 1e-2 and old.last_rank_mu_error() < 1e-8
    if acq == "ei":
        assert new.last_prefix_survivors() <= 16384     # EI is decided by the mean: the prefix bound prunes (PI, bounded by 1 wherever
                                                        # the improvement is positive, may not — it then takes the full pass, or three products)
    print(f"\nN={N} M={M} D={D} {kind}/{acq}: prefix survivors {new.last_prefix_survivors()}, survivors new {new.last_contenders()} old {old.last_contenders()}, "
          f"rank err var {new.last_rank_error():.2e} / {old.last_rank_error():.2e}, mu {new.last_rank_mu_error():.2e}")
    parts = [new.ask(Xc[s:s + 7000], global_offset=s) for s in range(0, M, 7000)]
    win = max(parts, key=lambda b: (b.value, -b.index))
    assert (win.index, win.value) == (bn.index, bn.value)
    for e in (new, old, slow, e64):
        e.close()


def _adversarial_grids(X, y, Xc):
    """Candidate orders that a first-wave calibration would not represent: sorted by distance to the incumbent, half of the
    rows duplicated (each duplicate right after its original), and a block-structured grid (discrete parameters)."""
    inc = X[int(np.argmin(y))]
    order = np.argsort(((Xc - inc) ** 2).sum(1))
    yield "sorted-near-first", Xc[order]
    yield "sorted-far-first", Xc[order[::-1]]
    half = Xc[: len(Xc) // 2]
    yield "half-duplicated", np.repeat(half, 2, axis=0)
    disc = Xc.copy()
    disc[:, : Xc.shape[1] // 2] = np.round(disc[:, : Xc.shape[1] // 2] * 3) / 3
    yield "discrete-blocks", disc[np.lexsort(disc[:, : Xc.shape[1] // 2].T[::-1])]


def test_ranking_pass_on_non_exchangeable_candidate_orders():
    """Stratified calibration: on sorted, duplicated and block-structured grids the ranking pass (both variants) returns
    bit for bit what the three-product sweep and the FP64 engine return."""
    N, M, D = 2048, 60000, 16
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    kw = dict(kind="matern52", acq="ei", **th)
    new = _engine(kw, "tc"); new.tell(X, y)
    old = _engine(kw, "tc", rank_tc=False); old.tell(X, y)
    slow = _engine(kw, "tc", tc_fast=False); slow.tell(X, y)
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    for name, G in _adversarial_grids(X, y, Xc):
        bn, bo, bs, b6 = new.ask(G), old.ask(G), slow.ask(G), e64.ask(G)
        assert _same(bn, bo) and _same(bn, bs) and (bo.index, bo.value) == (bs.index, bs.value), name
        assert bn.index == b6.index and abs(bn.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value)), name
        print(f"\n{name}: index {bn.index} prefix survivors {new.last_prefix_survivors()} survivors {new.last_contenders()} rank err {new.last_rank_error():.2e} mu {new.last_rank_mu_error():.2e}")
    for e in (new, old, slow, e64):
        e.close()


def test_ranking_pass_on_a_flat_landscape_falls_back_and_still_decides_in_fp64():
    """A near-flat EI landscape (a 1e-4 cube around the incumbent: EI positive and equal to ~1e-6 across the grid): the prefix
    bound cannot prune (> 16384 survive), the full ranking pass cannot either (> 4096), the sweep is redone with three products,
    whose own window overflows too and is narrowed — the suggestion is still the FP64 engine's to the contract's tolerance and
    the caller can see how it was decided."""
    N, M, D = 1024, 30000, 6
    X, y, _ = O.synthetic(N, 10, D)
    th = O.theta_of_record(D)
    r = np.random.default_rng(5)
    G = np.clip(X[int(np.argmin(y))] + 0.02 + 1e-4 * (r.random((M, D)) - 0.5), 0, 1)
    kw = dict(kind="matern52", acq="ei", **th)
    new = _engine(kw, "tc"); new.tell(X, y)
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    bn, b6 = new.ask(G), e64.ask(G)
    print(f"\nflat: prefix survivors {new.last_prefix_survivors()} contenders {new.last_contenders()} decision {new.last_unrefined()} value {bn.value:.3e}")
    assert new.last_prefix_survivors() > 16384 and new.last_contenders() > 4096 and new.last_unrefined() in (1, 2) and b6.value > 1e-6
    ref = O.suggest(X, y, G, kind="matern52", acq="ei", **th)
    assert abs(bn.value - ref["value"]) <= TOL_TC
    assert bn.index == b6.index or abs(ref["acq"][bn.index] - ref["value"]) <= TOL_TC
    new.close(); e64.close()


def test_cfg3_full_size_path_of_record():
    """BASELINE.json config 3 at full size through the path the bench times (array-free tensor-core sweep): N=8192, D=32,
    M=1,048,576, Matérn-5/2, EI.  The suggestion must be the FP64 engine's (same index, value to rounding) and the oracle's
    value on the winner row and on a 4096-row sample must agree to 1e-5 with the winner dominating the sample.  Every row of this
    grid, every acquisition and gp_hedge against an FP64 posterior of the whole grid: test_gpu_grid_scale.py."""
    N, M, D = 8192, 1_048_576, 32
    X, y, _ = O.synthetic(N, 1, D)
    Xc = np.random.default_rng(4321).random((M, D)).astype(np.float32)
    th = O.theta_of_record(D)
    kw = dict(kind="matern52", acq="ei", **th)
    xc = torch.tensor(Xc, device="cuda")
    new = _engine(kw, "tc"); new.tell(X, y)
    bn = new.ask(xc)
    surv, rerr, merr, psurv = new.last_contenders(), new.last_rank_error(), new.last_rank_mu_error(), new.last_prefix_survivors()
    assert new.last_unrefined() == 0 and 1 <= psurv <= 16384
    full = _engine(kw, "tc", rank_prefix=0); full.tell(X, y)
    bf = full.ask(xc)
    assert _same(bf, bn) and full.last_prefix_survivors() == -1
    full.close()
    old = _engine(kw, "tc", rank_tc=False); old.tell(X, y)
    bo = old.ask(xc)
    old.close()
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    b6 = e64.ask(xc)
    e64.close()
    assert _same(bn, bo)
    assert bn.index == b6.index and abs(bn.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value))
    sample = np.concatenate([[bn.index], np.random.default_rng(9).choice(M, 4096, replace=False)])
    fit = O.gp_fit(X, y, kind="matern52", **{k: th[k] for k in ("length_scale", "amplitude", "noise")})
    mu, std = O.gp_predict(fit, Xc[sample].astype(np.float64))
    a = O.acquisition(mu, std, float(y.min()), "ei", th["xi"], th["kappa"])
    print(f"\ncfg3 full size: index {bn.index} value {bn.value:.10f} oracle {a[0]:.10f} |d|={abs(bn.value - a[0]):.2e} prefix survivors {psurv} survivors {surv} "
          f"rank err var {rerr:.2e} mu {merr:.2e} next best of sample {np.max(a[1:]):.4f}")
    assert abs(bn.value - a[0]) <= TOL_TC
    assert a[0] >= np.max(a[1:])
    new.close()


@pytest.mark.parametrize("N,D,kind", [(700, 5, "matern52"), (2048, 16, "rbf"), (65, 3, "matern52")])
def test_lml_batch_matches_one_fit_per_theta_and_the_oracle(N, D, kind):
    """kbo_lml_batch: G factorisations on G streams (SURVEY.md §8(f)1).  Each value equals what a full fit at that θ reports
    (and the oracle's $SK/_gpr.py:604-618 restatement); a θ whose Gram matrix is not positive definite reads −inf; ARD length
    scales work; the handle's fitted state is untouched; 8 θ cost a small multiple of one fit."""
    import time
    X, y, Xc = O.synthetic(N, 100, D)
    th = O.theta_of_record(D)
    eng = _engine(dict(kind=kind, acq="ei", **th), "f64")
    eng.tell(X, y)
    before = eng.ask(Xc)
    thetas = [dict(length_scale=th["length_scale"] * m, noise=nz) for m, nz in ((0.25, 1e-3), (0.5, 1e-2), (1.0, 1e-3), (1.0, 1e-6), (2.0, 1e-3),
                                                                               (4.0, 1e-1), (0.7, 3e-4))]
    thetas.append(dict(length_scale=np.linspace(0.5, 2.0, D) * th["length_scale"], noise=1e-3))       # anisotropic
    got = eng.lml_batch(X, y, thetas)
    for t, g in zip(thetas, got):
        one = _engine(dict(kind=kind, acq="ei", **{**th, **t}), "f64")
        one.tell(X, y)
        ref = one.fit_info()["lml"]
        orc = O.gp_fit(X, y, kind=kind, length_scale=t["length_scale"], amplitude=th["amplitude"], noise=t["noise"])["lml"]
        assert abs(g - ref) <= 1e-9 * max(1.0, abs(ref)), (t, g, ref)
        assert abs(g - orc) <= 1e-7 * max(1.0, abs(orc)), (t, g, orc)
        one.close()
    after = eng.ask(Xc)
    assert (before.index, before.value) == (after.index, after.value)
    # duplicate rows with zero noise: not positive definite -> -inf for that θ only
    Xd, yd = np.concatenate([X, X[:1]]), np.concatenate([y, y[:1]])
    got = eng.lml_batch(Xd, yd, [dict(noise=0.0), dict(noise=1e-3)])
    assert got[0] == -np.inf and np.isfinite(got[1])
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(3):
        eng.lml_batch(X, y, thetas)
    torch.cuda.synchronize(); tb = (time.perf_counter() - t0) / 3
    t0 = time.perf_counter()
    for _ in range(3):
        eng.tell(X, y)
    torch.cuda.synchronize(); t1 = (time.perf_counter() - t0) / 3
    print(f"\nN={N}: lml_batch of {len(thetas)} thetas {tb * 1e3:.2f} ms, one fit {t1 * 1e3:.2f} ms (ratio {tb / t1:.2f})")
    eng.close()


@pytest.mark.parametrize("N,M,D,kind,acq", [(2048, 30000, 32, "matern52", "ei"), (3000, 20000, 12, "matern52", "lcb"), (2600, 25000, 8, "rbf", "ei")])
def test_lazy_inverse_sweep_matches_the_full_fit(N, M, D, kind, acq):
    """kbo_set_lazy_inverse (default): a tensor-core fit forms only the leading rows of W; alpha, the survivors' exact variances
    and the lower bound on the maximum come from panel solves with L and from the sigma -> 0 limit.  The suggestion must equal
    the eager fit's (W formed) and the FP64 engine's to FP64 rounding; everything that needs all of W (arrays, append, LML
    gradient, state) still works afterwards and agrees with the eager engine."""
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    kw = dict(kind=kind, acq=acq, **th)
    lazy = _engine(kw, "tc"); lazy.tell(X, y)
    eager = _engine(kw, "tc", lazy_inverse=False); eager.tell(X, y)
    e64 = _engine(kw, "f64"); e64.tell(X, y)
    il, ie = lazy.fit_info(), eager.fit_info()
    assert abs(il["lml"] - ie["lml"]) <= 1e-9 * max(1.0, abs(ie["lml"]))       # alpha by solves vs Wᵀ(W yn)
    bl, be, b6 = lazy.ask(Xc), eager.ask(Xc), e64.ask(Xc)
    print(f"\\nN={N} {kind}/{acq}: lazy kept {lazy.last_prefix_survivors()} (decided among {lazy.last_contenders()}), eager kept {eager.last_prefix_survivors()}")
    assert bl.index == be.index == b6.index
    assert abs(bl.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value)) and abs(bl.value - be.value) <= 1e-10 * max(1.0, abs(be.value))
    assert abs(bl.mu - b6.mu) <= 1e-9 and abs(bl.std - b6.std) <= 1e-8
    assert lazy.last_unrefined() == 0
    # consumers of the whole inverse after a lazy fit
    for a_, b_ in zip(lazy.state(), eager.state()):
        np.testing.assert_allclose(a_.cpu().numpy(), b_.cpu().numpy(), rtol=0, atol=5e-10)
    gl, ge = lazy.lml_grad()[1], eager.lml_grad()[1]
    np.testing.assert_allclose(gl, ge, rtol=1e-8, atol=1e-8)
    _, _, _, al = lazy.ask(Xc[:3000], return_arrays=True)
    _, _, _, ae = eager.ask(Xc[:3000], return_arrays=True)
    np.testing.assert_allclose(al.cpu().numpy(), ae.cpu().numpy(), rtol=0, atol=1e-9)
    lazy.tell(X[:N - 2], y[:N - 2]); eager.tell(X[:N - 2], y[:N - 2])             # lazy again, then append forms W
    for i in (N - 2, N - 1):
        lazy.append(X[i], y[i]); eager.append(X[i], y[i])
    b2l, b2e = lazy.ask(Xc), eager.ask(Xc)
    assert b2l.index == b2e.index and abs(b2l.value - b2e.value) <= 1e-9
    for e in (lazy, eager, e64):
        e.close()


@pytest.mark.parametrize("N,M,D,mode", [(700, 5000, 5, "tc"), (2304, 20000, 16, "tc"), (1500, 4000, 7, "f64")])
def test_fit_variants_agree(N, M, D, mode, tmp_path):
    """The factorisation's schedules — v3 (default: diagonal-block chain on its own SM partition, near / far shadows, look-ahead
    depth 3 with merged bulk updates), the same on plain priority streams, and the one-stream sequence (kbo_potrf, kbo_trtri) — are
    the same arithmetic up to the order the trailing updates are applied in: L, W, alpha, LML and the suggestion agree to FP64
    rounding, and all of them with the oracle's Cholesky."""
    import os, subprocess, sys
    runs = {}
    for name, env in (("v3", {}), ("v3-unpartitioned", {"KBO_FIT_NO_PARTITION": "1"}), ("serial", {"KBO_FIT_SERIAL": "1"})):
        out = str(tmp_path / f"{name}.npz")
        subprocess.run([sys.executable, os.path.join(os.path.dirname(__file__), "_fit_variant.py"), str(N), str(M), str(D), mode, out],
                       check=True, env={**os.environ, **env}, timeout=300)
        runs[name] = np.load(out)
    X, y, _ = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    fit = O.gp_fit(X, y, kind="matern52", length_scale=th["length_scale"], amplitude=th["amplitude"], noise=th["noise"])
    ref = runs["serial"]
    scale = np.abs(fit["L"]).max()
    assert np.abs(np.tril(ref["L"]) - fit["L"]).max() <= 1e-11 * scale
    for name, r in runs.items():
        assert np.abs(np.tril(r["L"]) - np.tril(ref["L"])).max() <= 1e-12 * scale, name
        assert np.abs(r["W"] - ref["W"]).max() <= 1e-9 * np.abs(ref["W"]).max(), name
        np.testing.assert_allclose(r["alpha"], ref["alpha"], rtol=0, atol=1e-9 * np.abs(ref["alpha"]).max(), err_msg=name)
        assert abs(float(r["lml"]) - float(ref["lml"])) <= 1e-10 * abs(float(ref["lml"])), name
        assert int(r["index"]) == int(ref["index"]) and abs(float(r["value"]) - float(ref["value"])) <= 1e-10 * max(1.0, abs(float(ref["value"]))), name


def test_fp64_kstar_kernel_gives_the_same_mean_for_few_and_many_rows():
    """With fewer CTAs than one wave the FP64 K* kernel splits the trial tiles over blockIdx.y and sums the partial means in split
    order: a candidate's mean must not depend (beyond FP64 rounding) on how many rows were swept with it."""
    N, M, D = 1500, 40000, 9
    X, y, Xc = O.synthetic(N, M, D)
    g = dict(kind="matern52", acq="ei", **O.theta_of_record(D))
    e = _engine(g, "f64"); e.tell(X, y)
    _, mu_all, sd_all, _ = e.ask(Xc, return_arrays=True)
    for rows in (1, 130, 3000):
        _, mu, sd, _ = e.ask(Xc[:rows], return_arrays=True)
        np.testing.assert_allclose(mu.cpu().numpy(), mu_all.cpu().numpy()[:rows], rtol=0, atol=1e-12 * max(1.0, float(mu_all.abs().max())))
        np.testing.assert_allclose(sd.cpu().numpy(), sd_all.cpu().numpy()[:rows], rtol=0, atol=1e-10)
    fit = O.gp_fit(X, y, kind="matern52", length_scale=g["length_scale"], amplitude=g["amplitude"], noise=g["noise"])
    mu_ref, _ = O.gp_predict(fit, Xc[:130])
    _, mu, _, _ = e.ask(Xc[:130], return_arrays=True)
    np.testing.assert_allclose(mu.cpu().numpy(), mu_ref, rtol=0, atol=1e-8)
    e.close()


def test_lazy_fit_decides_among_hundreds_of_survivors_by_triangular_solves():
    """A lazy fit evaluates up to 256 survivors of the prefix bound in FP64 by cooperative panel solves with L (up to 64 right-hand
    sides per launch) instead of forming the rest of L^-1.  LCB with a growing kappa loosens the prefix bound: whatever the
    number of survivors — a handful, hundreds, or more than the cap (then the eager path runs) — the suggestion is the FP64
    engine's, and a candidate's value does not depend on how many survivors it was evaluated with (sharded asks are bit-equal)."""
    N, M, D = 2048, 30000, 32
    X, y, Xc = O.synthetic(N, M, D)
    th = O.theta_of_record(D)
    seen = []
    for kappa in (1.96, 6.0, 12.0, 20.0, 40.0):
        kw = dict(kind="matern52", acq="lcb", **{**th, "kappa": kappa})
        lazy = _engine(kw, "tc"); lazy.tell(X, y)
        e64 = _engine(kw, "f64"); e64.tell(X, y)
        bl, b6 = lazy.ask(Xc), e64.ask(Xc)
        seen.append(lazy.last_prefix_survivors())
        assert bl.index == b6.index and abs(bl.value - b6.value) <= 1e-10 * max(1.0, abs(b6.value)), (kappa, seen)
        assert lazy.last_unrefined() == 0
        if 1 <= seen[-1] <= 256:
            lazy.tell(X, y)     # a fresh lazy fit: the sharded asks below must not inherit a W formed by a fallback
            parts = [lazy.ask(Xc[s0:s0 + 10000], global_offset=s0) for s0 in range(0, M, 10000)]
            win = max(parts, key=lambda b: (b.value, -b.index))
            assert (win.index, win.value) == (bl.index, bl.value), (kappa, seen)
        lazy.close(); e64.close()
    print(f"\nprefix survivors by kappa: {seen}")
    assert any(64 < n <= 256 for n in seen), seen


def test_fit_is_bit_reproducible_run_to_run():
    """The default factorisation runs on a dozen streams ordered by events only; every read-modify-write of a block is ordered, so
    repeated fits of the same history must give bit-identical L, alpha and suggestion (a missing dependency shows up here as run-to-run
    differences long before it shows up as a wrong answer)."""
    N, M, D = 6144, 20000, 24
    X, y, Xc = O.synthetic(N, M, D)
    g = dict(kind="matern52", acq="ei", **O.theta_of_record(D))
    e = _engine(g, "tc")
    ref = None
    for it in range(5):
        e.tell(X, y)
        b = e.ask(Xc)
        Lm, _, al = e.state()
        cur = (Lm.clone(), al.clone(), b.index, b.value)
        if ref is None:
            ref = cur
        else:
            assert torch.equal(torch.tril(cur[0]), torch.tril(ref[0])), it
            assert torch.equal(cur[1], ref[1]), it
            assert (cur[2], cur[3]) == (ref[2], ref[3]), it
    e.close()
