"""CPU: the ENAS oracle's hand-written gradients against torch.autograd on an independent float64 restatement of the loss, and
hand-worked cases (nll = 0 with one op and one layer, the baseline recurrence, one Adam step, the arc length)."""
import itertools

import numpy as np
import pytest
import torch

from oracle import enas_oracle as O


def torch_loss(P, L, st, arc, adv, skc):
    """adv·nll + skc·Σ_{l>=1} kl_l for a fixed arc, written from the controller's definition (no shared code with the oracle)."""
    W, ge, we, ws, w1, w2, v = (P[n] for n in O.PARAM_NAMES)
    H = ge.shape[1]
    tgt = torch.tensor([1.0 - st["skip_target"], st["skip_target"]], dtype=torch.float64)

    def shp(z):
        if st["temperature"] is not None:
            z = z / st["temperature"]
        if st["tanh_const"] is not None:
            z = st["tanh_const"] * torch.tanh(z)
        return z

    def cell(x, c, h):
        z = torch.cat([x, h]) @ W
        i, f, o, g = torch.sigmoid(z[:H]), torch.sigmoid(z[H:2 * H]), torch.sigmoid(z[2 * H:3 * H]), torch.tanh(z[3 * H:])
        c = i * g + f * c
        return c, o * torch.tanh(c)

    c = h = torch.zeros(H, dtype=torch.float64)
    x = ge[0]
    nll = torch.zeros((), dtype=torch.float64)
    kl = torch.zeros((), dtype=torch.float64)
    anchors, aw = [], []
    for l in range(L):
        pos = l * (l + 1) // 2
        c, h = cell(x, c, h)
        op = int(arc[pos])
        nll = nll - torch.log_softmax(shp(h @ ws), 0)[op]
        c, h = cell(we[op], c, h)
        if l > 0:
            sk = []
            for j in range(l):
                q = torch.tanh(aw[j] + h @ w2) @ v[:, 0]
                s = shp(torch.stack([-q, q]))
                b = int(arc[pos + 1 + j])
                nll = nll - torch.log_softmax(s, 0)[b]
                g = torch.sigmoid(s)
                kl = kl + (g * torch.log(g / tgt)).sum()
                sk.append(b)
            x = sum((b * a for b, a in zip(sk, anchors)), torch.zeros(H, dtype=torch.float64)) / (1.0 + sum(sk))
        else:
            x = ge[0]
        anchors.append(h)
        aw.append(h @ w1)
    return adv * nll + skc * kl


def _check(L, H, n_ops, st, seed=0):
    rng = np.random.default_rng(seed + 1000 * L + 10 * H + n_ops)
    P = O.init_params(H, n_ops, rng)
    P = {n: a * 5 for n, a in P.items()}                  # larger weights: saturating gates and shaped logits away from 0
    arc = O.forward(P, L, st, uniforms=rng.random(L * (L + 1) // 2))["arc"]
    adv, skc = 0.7, 0.3
    G = O.backward(P, O.forward(P, L, st, arc=arc)["cache"], adv, skc)
    T = {n: torch.tensor(P[n], dtype=torch.float64, requires_grad=True) for n in O.PARAM_NAMES}
    torch_loss(T, L, st, arc, adv, skc).backward()
    for n in O.PARAM_NAMES:
        ref = T[n].grad.numpy() if T[n].grad is not None else np.zeros_like(P[n])   # unused at L = 1
        err = np.abs(G[n] - ref).max()
        assert err <= 1e-12 * max(1.0, np.abs(ref).max()), (n, err)


@pytest.mark.parametrize("L,H,n_ops", list(itertools.product((1, 2, 5, 12), (1, 8, 64), (1, 2, 7, 78))))
def test_gradients_equal_autograd(L, H, n_ops):
    _check(L, H, n_ops, O.settings())


@pytest.mark.parametrize("none", [("temperature",), ("tanh_const",), ("temperature", "tanh_const"), ("entropy_weight", "skip_weight")])
def test_gradients_equal_autograd_with_none_settings(none):
    st = O.settings(**{k: None for k in none})
    for L, H, n_ops in ((5, 8, 7), (12, 64, 78)):
        _check(L, H, n_ops, st, seed=7)


def test_one_op_one_layer_has_zero_nll():
    rng = np.random.default_rng(0)
    P = O.init_params(8, 1, rng)
    fw = O.forward(P, 1, O.settings(), uniforms=rng.random(1))
    assert fw["nll"] == 0.0 and fw["ent"] == 0.0 and list(fw["arc"]) == [0] and fw["kl"] == []


def test_arc_length_is_triangular():
    rng = np.random.default_rng(1)
    P = O.init_params(4, 3, rng)
    for L in (1, 2, 3, 7):
        fw = O.forward(P, L, O.settings(), uniforms=rng.random(L * (L + 1) // 2))
        assert len(fw["arc"]) == L * (L + 1) // 2
        assert [len(x) for x in O.organise_arc(fw["arc"], L)] == list(range(1, L + 1))


def test_baseline_recurrence_and_one_adam_step():
    rng = np.random.default_rng(2)
    st = O.settings(baseline_decay=0.9, learning_rate=0.01, entropy_weight=0.5)
    L, H, n_ops = 3, 4, 5
    P0 = O.init_params(H, n_ops, rng)
    s = O.new_state(P0)
    s["baseline"] = 0.25
    arc = O.forward(P0, L, st, uniforms=rng.random(6))["arc"]
    out = O.train_step(s, L, st, 2.0, arc=arc)
    r = 2.0 + 0.5 * out["ent"]
    assert out["baseline"] == pytest.approx(0.25 - 0.1 * (0.25 - r), abs=1e-15)
    lr_t = 0.01 * np.sqrt(1 - 0.999)
    for n in O.PARAM_NAMES:
        g = out["grads"][n]
        want = P0[n] - lr_t * g / (np.sqrt(0.001 * g * g) + 1e-3)
        np.testing.assert_allclose(s["params"][n], want, rtol=0, atol=1e-15)
        np.testing.assert_array_equal(s["m"][n], g)
    assert s["step"] == 1
    assert out["loss"] == pytest.approx(out["nll"] * (r - out["baseline"]) + 0.8 * np.mean(O.forward(P0, L, st, arc=arc)["kl"]))


def test_draw_takes_first_bin_past_u():
    p = np.array([0.25, 0.0, 0.5, 0.25])
    assert [O.draw(p, u) for u in (0.0, 0.2499, 0.25, 0.7499, 0.75, 0.999999)] == [0, 0, 2, 2, 3, 3]


def test_draw_falls_back_to_the_last_bin_with_weight():
    assert O.draw(np.array([0.5, 0.5, 0.0]), 1.0) == 1
