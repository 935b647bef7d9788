"""GPU: CMA-ES generation (kbo_cma_*) against the NumPy oracle.  The eigenbasis of C is only defined up to sign/order, so
parity is stated on basis-independent quantities: the oracle is fed the GPU's own steps Y and must reproduce mean, sigma,
C and both evolution paths after every generation; the eigendecomposition is checked by B·diag(d²)·Bᵀ = C, BᵀB = I.
Tolerances are relative to each quantity's own scale.  Long runs, ranking edge cases and the sampler: test_gpu_cma_long.py."""
import numpy as np
import pytest
import torch

from oracle import cma_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("D,lam", [(1, 4), (2, 6), (4, 8), (5, 8), (16, 32), (37, 50), (64, 255), (65, 257), (127, 1025),
                                   (128, 256), (128, 1024), (128, 4096), (128, 4097), (128, 8192)])
def test_generation_update_matches_oracle(D, lam):
    from kubeflow_b200.cmaes import CmaEs
    r = np.random.default_rng(D * 1000 + lam)
    m0 = r.uniform(-2, 2, D)
    es = CmaEs(m0, 1.3, popsize=lam, seed=5)
    ref = O.CmaState(m0, 1.3, lam)
    gens = 6 if lam <= 256 else 3
    for g in range(gens):
        z = torch.tensor(r.standard_normal((lam, D)), device="cuda")
        X = es.ask(z).cpu().numpy()
        st = es.state(with_Y=True)
        # ask: x = m + sigma*y with y ~ N(0, C): check against the oracle's own transform through C (basis-free)
        np.testing.assert_allclose(X, st["mean"] + st["sigma"] * st["Y"], atol=1e-12 * np.abs(X).max())
        Bm, d = st["B"], st["d"]
        np.testing.assert_allclose(Bm @ np.diag(d * d) @ Bm.T, ref.C, rtol=0, atol=1e-10 * np.linalg.norm(ref.C, 2))
        np.testing.assert_allclose(Bm.T @ Bm, np.eye(D), atol=1e-11)
        np.testing.assert_allclose(st["Y"], (z.cpu().numpy() * d) @ Bm.T, rtol=0, atol=1e-11 * np.abs(st["Y"]).max())
        f = O.rastrigin(X) if g % 2 else O.sphere(X)
        if g == 1:
            f[lam // 2] = f[lam - 1]         # a tie: lower sample index ranks first
        es.tell(f)
        O.tell(ref, st["Y"], f, znorm2=(z.cpu().numpy() ** 2).sum(1))
        got = es.state()
        np.testing.assert_allclose(got["mean"], ref.mean, rtol=0, atol=1e-11 * np.linalg.norm(ref.mean))
        assert abs(got["sigma"] - ref.sigma) < 1e-11 * ref.sigma
        np.testing.assert_allclose(got["C"], ref.C, rtol=0, atol=1e-11 * np.linalg.norm(ref.C, 2))
        np.testing.assert_allclose(got["p_sigma"], ref.p_sigma, rtol=0, atol=1e-10 * np.linalg.norm(ref.p_sigma))
        np.testing.assert_allclose(got["pc"], ref.pc, rtol=0, atol=1e-10 * np.linalg.norm(ref.pc))
        assert got["generation"] == g + 1
    es.close()


def test_builtin_sampler_statistics_and_convergence():
    from kubeflow_b200.cmaes import CmaEs
    es = CmaEs(np.zeros(64), 1.0, popsize=8192, seed=123)
    X = es.ask().cpu().numpy()
    assert abs(X.mean()) < 0.01 and abs(X.std() - 1.0) < 0.01              # N(0, I) before any update
    assert abs(np.corrcoef(X[:, 0], X[:, 1])[0, 1]) < 0.05
    X2 = es.ask().cpu().numpy()
    assert np.array_equal(X, X2)                                          # same (seed, generation) → same stream
    es.close()
    es = CmaEs(np.full(24, 3.0), 2.0, popsize=48, seed=1)
    out = es.run_synthetic("sphere", 300)
    assert out["best_f"] < 1e-10, out
    es.close()


def test_cfg4_shape_runs_and_improves():
    from kubeflow_b200.cmaes import CmaEs
    es = CmaEs(np.full(128, 3.0), 2.0, popsize=4096, seed=7)
    out = es.run_synthetic("rastrigin", 200)
    print("\ncfg4 CMA-ES D=128 lambda=4096 200 generations:", out)
    assert out["best_f"] < 10 * 128 + 9 * 128 and out["generations_per_s"] > 100
    st = es.state()
    assert np.linalg.eigvalsh(st["C"]).min() > 0
    es.close()


def test_cma_errors():
    from kubeflow_b200 import _lib as Lb
    from kubeflow_b200.cmaes import CmaEs
    with pytest.raises(Lb.KboInvalidArgument):
        CmaEs(np.zeros(129), 1.0, popsize=16)
    with pytest.raises(Lb.KboInvalidArgument):
        CmaEs(np.zeros(4), -1.0, popsize=16)
    es = CmaEs(np.zeros(4), 1.0, popsize=8)
    with pytest.raises(Lb.KboError):
        es.tell(np.zeros(8))          # tell before ask
    es.close()
