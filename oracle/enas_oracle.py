"""FP64 NumPy restatement of Katib's ``enas`` suggestion: the macro-search LSTM controller of ENAS, its REINFORCE training step
and its architecture draws (test-only; the GPU engine is kubeflow_b200/csrc/enas.cu).

Katib's ENAS source (``pkg/suggestion/v1beta1/nas/enas/``: Controller.py, Operation.py, AlgorithmSettings.py, service.py) is
not available here; every rule below is restated from memory of upstream and marked [RECALL].

Controller [RECALL]: parameters w_lstm (2H × 4H, no bias), g_emb (1 × H), w_emb (n_ops × H), w_soft (H × n_ops), w_attn_1,
w_attn_2 (H × H), v_attn (H × 1), all U(-0.1, 0.1).  LSTM cell: [i f o g] = [x, h]·w_lstm; i, f, o = σ, g = tanh;
c' = i⊙g + f⊙c; h' = o⊙tanh(c').  Logit shaping s(z) = tanh_const·tanh(z / temperature), a factor skipped when its setting is
None.  Per layer l: cell, op ~ softmax(s(h·w_soft)), input = w_emb[op], cell; for l > 0 and each j < l,
q_j = tanh(a_j·w_attn_1 + h·w_attn_2)·v_attn, skip_j ~ softmax(s([-q_j, q_j])), kl_l = Σ_j Σ_b σ(s_b)·log(σ(s_b) / t_b) with
t = (1 - skip_target, skip_target) (upstream's elementwise sigmoid, kept), input = Σ_j skip_j·a_j / (1 + Σ_j skip_j); for
l = 0 input = g_emb; the anchor a_l = h.  nll sums the cross-entropies of every decision; ent sums the stop-gradient terms
CE·exp(-CE).

Training step [RECALL]: r = R + entropy_weight·ent; baseline ← baseline - (1 - baseline_decay)(baseline - r);
loss = nll·(r - baseline) + skip_weight·mean_{l>=1} kl_l (0 for L = 1, where upstream's mean is over no layer); TF Adam with
β1 = 0, β2 = 0.999, ε̂ = 1e-3: lr_t = lr·sqrt(1 - β2^t), θ -= lr_t·m / (sqrt(v) + ε̂), t over the controller's life.
Departure, stated once: upstream wraps lr in a staircase exponential decay whose first decay step no Experiment reaches; the
rate here is constant.  None for entropy_weight or skip_weight drops that term (the same as 0).

Draws (this engine's rule, not upstream's multinomial): a decision takes the first bin whose cumulative probability exceeds
the uniform u.

Search space [RECALL: Operation.py] and reply [RECALL: service.py], restated here independently of the service: ``expand``
and ``reply_strings`` below.
The settings' defaults are recalled [RECALL: AlgorithmSettings.py]; their accepted ranges (hidden size and step counts >= 1,
temperature and tanh_const > 0, entropy and skip weights >= 0, baseline_decay in [0, 1], learning_rate in (0, 1],
skip_target in (0, 1), and "None" for the four that upstream allows to be None) are guesses, as are the nas_config checks.
"""
from __future__ import annotations

import itertools
import json

import numpy as np

from kubeflow_b200.suggestion import api_pb as api

PARAM_NAMES = ("w_lstm", "g_emb", "w_emb", "w_soft", "w_attn_1", "w_attn_2", "v_attn")
STAT_NAMES = ("nll", "ent", "kl", "loss", "baseline", "skip_rate")


def settings(**kw) -> dict:
    """Controller settings with upstream's defaults (keys as in kubeflow_b200.enas.DEFAULT_SETTINGS)."""
    st = dict(temperature=5.0, tanh_const=2.25, entropy_weight=1e-5, baseline_decay=0.999, learning_rate=5e-5, skip_target=0.4,
              skip_weight=0.8)
    st.update(kw)
    return st


def init_params(H: int, n_ops: int, rng) -> dict:
    u = lambda *s: rng.uniform(-0.1, 0.1, s)
    return dict(w_lstm=u(2 * H, 4 * H), g_emb=u(1, H), w_emb=u(n_ops, H), w_soft=u(H, n_ops), w_attn_1=u(H, H), w_attn_2=u(H, H),
                v_attn=u(H, 1))


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def shape(st, z):
    if st["temperature"] is not None:
        z = z / st["temperature"]
    if st["tanh_const"] is not None:
        z = st["tanh_const"] * np.tanh(z)
    return z


def dshape(st, z):
    d = np.ones_like(np.asarray(z, dtype=np.float64))
    if st["temperature"] is not None:
        z = z / st["temperature"]
        d = d / st["temperature"]
    if st["tanh_const"] is not None:
        d = d * st["tanh_const"] * (1.0 - np.tanh(z) ** 2)
    return d


def _softmax(s):
    e = np.exp(s - s.max())
    return e / e.sum()


def philox_uniform(seed: int, draw_counter: int, arc: int, decision: int) -> float:
    """The engine's uniform of a decision: word 0 of Philox4x32-10 at counter (draw counter lo, hi, arc, decision), key
    (seed lo, hi), as (word >> 8)·2^-24 (kbo.h)."""
    M = 0xFFFFFFFF
    c0, c1, c2, c3 = draw_counter & M, (draw_counter >> 32) & M, arc & M, decision & M
    k0, k1 = seed & M, (seed >> 32) & M
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M, p1 & M, ((p0 >> 32) ^ c3 ^ k1) & M, p0 & M
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return (c0 >> 8) * 2.0 ** -24


def draw(p, u: float) -> int:
    """The first bin whose cumulative probability exceeds u; when rounding leaves u at or above the total, the last bin
    with nonzero probability."""
    c = np.cumsum(p)
    i = int(np.searchsorted(c, u, side="right"))
    return i if i < len(p) else int(np.flatnonzero(np.asarray(p) > 0)[-1])


def expand(operations) -> list:
    """[RECALL: Operation.py] One (opt_type, {param: value}) per operation id: each operation's specs as value lists
    (INT range(min, max + 1, step); DOUBLE np.arange(min, max + step, step) without an endpoint above max; CATEGORICAL the list
    as strings), combined by itertools.product in spec order, operations in order."""
    out = []
    for op in operations:
        names, lists = [], []
        for p in op.parameter_specs.parameters:
            fs = p.feasible_space
            if p.parameter_type == api.INT:
                v = list(range(int(fs.min), int(fs.max) + 1, int(fs.step)))
            elif p.parameter_type == api.DOUBLE:
                d = np.arange(float(fs.min), float(fs.max) + float(fs.step), float(fs.step))
                v = [float(x) for x in (d[:-1] if d[-1] > float(fs.max) else d)]
            else:
                v = list(fs.list)
            names.append(p.name)
            lists.append(v)
        out += [(op.operation_type, dict(zip(names, combo))) for combo in itertools.product(*lists)]
    return out


def organise_arc(arc, L: int) -> list:
    """The flat arc per layer: layer l holds its op and l skip bits."""
    layers, i = [], 0
    for l in range(L):
        layers.append([int(x) for x in arc[i:i + l + 1]])
        i += l + 1
    return layers


def reply_strings(arc, L: int, input_sizes, output_sizes, expanded) -> tuple:
    """[RECALL: service.py] (architecture, nn_config) of one flat arc: the arc per layer, and num_layers, input_sizes,
    output_sizes and the embedding of the distinct ops in layer order, each json.dumps'd with " replaced by '."""
    layers = organise_arc(arc, L)
    emb = {}
    for layer in layers:
        t, params = expanded[layer[0]]
        emb.setdefault(str(layer[0]), {"opt_id": layer[0], "opt_type": t, "opt_params": params})
    cfg = {"num_layers": L, "input_sizes": list(input_sizes), "output_sizes": list(output_sizes), "embedding": emb}
    return json.dumps(layers).replace('"', "'"), json.dumps(cfg).replace('"', "'")


def boundary_distance(p, u: float, i: int) -> float:
    """Distance from u to the nearer CDF boundary of bin i."""
    c = np.concatenate([[0.0], np.cumsum(p)])
    return float(min(abs(u - c[i]), abs(u - c[i + 1])))


def _cell(W, x, c, h):
    H = h.shape[0]
    xh = np.concatenate([x, h])
    z = xh @ W
    i, f, o, g = _sig(z[:H]), _sig(z[H:2 * H]), _sig(z[2 * H:3 * H]), np.tanh(z[3 * H:])
    cn = i * g + f * c
    hn = o * np.tanh(cn)
    return cn, hn, dict(xh=xh, c=c, cn=cn, i=i, f=f, o=o, g=g)


def forward(P: dict, L: int, st: dict, arc=None, uniforms=None) -> dict:
    """One pass of the sampler.  ``arc`` imposes the decisions (teacher forcing); otherwise ``uniforms`` (L(L+1)/2) draw them.
    Returns arc, nll, ent, kl (list over layers l >= 1), the per-decision probabilities and the cache of the backward pass."""
    H = P["g_emb"].shape[1]
    tgt = np.array([1.0 - st["skip_target"], st["skip_target"]])
    c, h, x = np.zeros(H), np.zeros(H), P["g_emb"][0].copy()
    cells, ops, op_z, op_p, att, anchors, aw1, skips_l, out = [], [], [], [], [], [], [], [], []
    nll = ent = 0.0
    kls, kls_abs, skip_p, margins = [], [], [], []
    for l in range(L):
        pos = l * (l + 1) // 2
        c, h, cell = _cell(P["w_lstm"], x, c, h)
        cells.append(cell)
        z = h @ P["w_soft"]
        s = shape(st, z)
        p = _softmax(s)
        if arc is not None:
            op = int(arc[pos])
        else:
            op = draw(p, float(uniforms[pos]))
            margins.append(boundary_distance(p, float(uniforms[pos]), op))
        ce = np.log(np.exp(s - s.max()).sum()) + s.max() - s[op]
        nll += ce
        ent += ce * np.exp(-ce)
        ops.append(op)
        op_z.append(z)
        op_p.append(p)
        out.append(op)
        x = P["w_emb"][op].copy()
        c, h, cell = _cell(P["w_lstm"], x, c, h)
        cells.append(cell)
        if l > 0:
            hw2 = h @ P["w_attn_2"]
            kl, kla, sk, rows = 0.0, 0.0, [], []
            for j in range(l):
                T = np.tanh(aw1[j] + hw2)
                q = float(T @ P["v_attn"][:, 0])
                s2 = shape(st, np.array([-q, q]))
                p2 = _softmax(s2)
                if arc is not None:
                    b = int(arc[pos + 1 + j])
                else:
                    b = draw(p2, float(uniforms[pos + 1 + j]))
                    margins.append(boundary_distance(p2, float(uniforms[pos + 1 + j]), b))
                ce = np.log(np.exp(s2 - s2.max()).sum()) + s2.max() - s2[b]
                nll += ce
                ent += ce * np.exp(-ce)
                g = _sig(s2)
                kl += float((g * np.log(g / tgt)).sum())
                kla += float(np.abs(g * np.log(g / tgt)).sum())
                sk.append(b)
                skip_p.append(p2[1])
                rows.append(dict(T=T, q=q, skip=b))
                out.append(b)
            kls.append(kl)
            kls_abs.append(kla)
            att.append(rows)
            skips_l.append(sk)
            x = sum(b * a for b, a in zip(sk, anchors)) / (1.0 + sum(sk))
        else:
            att.append([])
            skips_l.append([])
            x = P["g_emb"][0].copy()
        anchors.append(h)
        aw1.append(h @ P["w_attn_1"])
    cache = dict(cells=cells, ops=ops, op_z=op_z, op_p=op_p, att=att, anchors=anchors, skips=skips_l, L=L, st=st)
    return dict(arc=np.array(out, dtype=np.int64), nll=nll, ent=ent, kl=kls, kl_abs=kls_abs, op_p=op_p, skip_p=np.array(skip_p), margins=margins,
                cache=cache)


def _cell_bwd(W, cell, dh, dc):
    i, f, o, g, c, cn = cell["i"], cell["f"], cell["o"], cell["g"], cell["c"], cell["cn"]
    tc = np.tanh(cn)
    dct = dc + dh * o * (1 - tc * tc)
    dz = np.concatenate([dct * g * i * (1 - i), dct * c * f * (1 - f), dh * tc * o * (1 - o), dct * i * (1 - g * g)])
    dW = np.outer(cell["xh"], dz)
    dxh = W @ dz
    H = dh.shape[0]
    return dW, dxh[:H], dxh[H:], dct * f


def backward(P: dict, cache: dict, adv: float, skc: float) -> dict:
    """Gradients of adv·nll + skc·Σ_{l>=1} kl_l with respect to every parameter (the sampled arc held fixed)."""
    st, L = cache["st"], cache["L"]
    H = P["g_emb"].shape[1]
    tgt = np.array([1.0 - st["skip_target"], st["skip_target"]])
    G = {n: np.zeros_like(P[n]) for n in PARAM_NAMES}
    W, W1, W2, v = P["w_lstm"], P["w_attn_1"], P["w_attn_2"], P["v_attn"][:, 0]
    cells, anchors = cache["cells"], cache["anchors"]
    dh, dc = np.zeros(H), np.zeros(H)
    gaw1 = [np.zeros(H) for _ in range(L)]      # gradient of anchor_l · w_attn_1
    da = [np.zeros(H) for _ in range(L)]        # gradient of anchor l through later inputs
    for l in range(L - 1, -1, -1):
        dhb = dh + da[l] + W1 @ gaw1[l]
        G["w_attn_1"] += np.outer(anchors[l], gaw1[l])
        if l > 0:
            du_sum = np.zeros(H)
            for j, row in enumerate(cache["att"][l]):
                q, T, b = row["q"], row["T"], row["skip"]
                zz = np.array([-q, q])
                s2 = shape(st, zz)
                p2 = _softmax(s2)
                g = _sig(s2)
                ds = adv * (p2 - np.eye(2)[b]) + skc * g * (1 - g) * (np.log(g / tgt) + 1.0)
                dz = ds * dshape(st, zz)
                dq = dz[1] - dz[0]
                G["v_attn"][:, 0] += dq * T
                du = dq * v * (1 - T * T)
                du_sum += du
                gaw1[j] += du
            G["w_attn_2"] += np.outer(anchors[l], du_sum)
            dhb = dhb + W2 @ du_sum
        dW, dx, dh_, dc = _cell_bwd(W, cells[2 * l + 1], dhb, dc)
        G["w_lstm"] += dW
        G["w_emb"][cache["ops"][l]] += dx
        z, p, op = cache["op_z"][l], cache["op_p"][l], cache["ops"][l]
        oh = np.zeros(len(p))
        oh[op] = 1.0
        dzs = adv * (p - oh) * dshape(st, z)
        hA = cells[2 * l + 1]["xh"][H:]
        G["w_soft"] += np.outer(hA, dzs)
        dh_ = dh_ + P["w_soft"] @ dzs
        dW, dx, dh, dc = _cell_bwd(W, cells[2 * l], dh_, dc)
        G["w_lstm"] += dW
        if l <= 1:
            G["g_emb"][0] += dx
        else:
            sk = cache["skips"][l - 1]
            for j, b in enumerate(sk):
                if b:
                    da[j] += dx / (1.0 + sum(sk))
    return G


def new_state(params: dict) -> dict:
    P = {n: np.asarray(params[n], dtype=np.float64).copy() for n in PARAM_NAMES}
    return dict(params=P, m={n: np.zeros_like(P[n]) for n in PARAM_NAMES}, v={n: np.zeros_like(P[n]) for n in PARAM_NAMES},
                baseline=0.0, step=0)


def train_step(state: dict, L: int, st: dict, R: float, arc=None, uniforms=None) -> dict:
    """One REINFORCE step in place on ``state``; returns the step's statistics and arc."""
    P = state["params"]
    fw = forward(P, L, st, arc=arc, uniforms=uniforms)
    ew = st["entropy_weight"] or 0.0
    sw = st["skip_weight"] or 0.0
    r = R + ew * fw["ent"]
    b = state["baseline"]
    b = b - (1.0 - st["baseline_decay"]) * (b - r)
    state["baseline"] = b
    adv = r - b
    klm = float(np.mean(fw["kl"])) if L > 1 else 0.0
    skc = sw / (L - 1) if L > 1 else 0.0
    G = backward(P, fw["cache"], adv, skc)
    state["step"] += 1
    lr_t = st["learning_rate"] * np.sqrt(1.0 - 0.999 ** state["step"])
    for n in PARAM_NAMES:
        g = G[n]
        state["m"][n] = g.copy()
        state["v"][n] = 0.999 * state["v"][n] + 0.001 * g * g
        P[n] -= lr_t * g / (np.sqrt(state["v"][n]) + 1e-3)
    npairs = L * (L - 1) // 2
    nskip = sum(sum(s) for s in fw["cache"]["skips"])
    # kl_abs: the mean over layers of Σ|terms| — the scale of kl's rounding when its terms cancel
    return dict(nll=fw["nll"], ent=fw["ent"], kl=klm, kl_abs=float(np.mean(fw["kl_abs"])) if L > 1 else 0.0, loss=fw["nll"] * adv + sw * klm, baseline=b,
                skip_rate=nskip / npairs if npairs else 0.0, arc=fw["arc"], grads=G)
