"""GPU: the tensor-core K* kernel's mean-only tiles (tc_kstar.cu).  A pruning pass stores only a prefix of the K* plane; the
tiles past it still feed the normalised mean μ̃.  A mean-only body that dropped or altered a tile would only inflate the
calibrated mean error, and the sweep would fall back to the slower path without any other test noticing.  So: μ̃ with a prefix
is bitwise μ̃ with every column stored, the stored prefix is bitwise the full plane's, and nothing past the prefix is written."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

POISON = -1024.0   # exactly representable in fp16, and no kernel value (those are >= 0)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32).cpu().numpy()


@pytest.mark.parametrize("kind", ["rbf", "matern52"])
@pytest.mark.parametrize("N,M,D", [(1000, 700, 7), (1000, 513, 100), (8192, 1300, 32), (8192, 300, 7)])
def test_kstar_prefix_store_leaves_mean_and_stored_columns_bit_identical(kind, N, M, D):
    from kubeflow_b200.gp import GPEngine
    X, y, Xc = O.synthetic(N, M, D)
    eng = GPEngine(0, kernel=kind, acq="ei", var_mode="tc", **O.theta_of_record(D))
    try:
        eng.tell(X, y)
        xc = torch.tensor(Xc.astype(np.float32), device="cuda")
        mu_full, plane_full = eng.kstar_pass(xc)
        npad = plane_full.shape[1]
        assert np.all(_bits(plane_full[:M, N:]) == 0), "padding columns of the full plane are not zero"
        # the production ranking pass runs the same kernel: its mean and plane are these
        mu_rk, _, plane_rk = eng.rank_pass(xc, 1, want_plane=True)
        assert np.array_equal(_bits(mu_rk), _bits(mu_full))
        assert np.array_equal(_bits(plane_rk), _bits(plane_full[:M]))
        for store_cols in (0, 300, 1024):
            stored = min(-(-store_cols // 128) * 128, npad)
            poisoned = torch.full_like(plane_full, POISON)
            mu_p, plane_p = eng.kstar_pass(xc, store_cols=store_cols, plane=poisoned)
            assert np.array_equal(_bits(mu_p), _bits(mu_full)), f"store_cols={store_cols}: mean differs from the full-store mean"
            assert np.array_equal(_bits(plane_p[:, :stored]), _bits(plane_full[:, :stored])), f"store_cols={store_cols}: stored prefix differs"
            rest = plane_p[:, stored:].float().cpu().numpy()
            assert np.all(rest == POISON), f"store_cols={store_cols}: {int(np.sum(rest != POISON))} entries past the prefix were written"
    finally:
        eng.close()
