"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the per-particle set transformer (tests/set_transformer_oracle.py) on sets
of different sizes: every set is padded to L = number_particles rows and set s has l_s real particles.  [KERAS] the attention is
Keras 2 MultiHeadAttention(..., attention_mask=mask[:, None, :]): masked scores get a large negative addend, so with at least
one real key their softmax weight is exactly 0 -- here they are -inf.  The mean over the particles is GlobalAveragePooling1D with
a mask (over the l_s real rows), the KL sums over the real particles.  Padding rows enter the encoder as zeros, get u = 0, a
zero attention output and zero gradients.  A hand-written reverse mode, a torch float64 autograd twin and a Model.fit loop on
ragged batches.  The product path never imports this module."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import dib_oracle as O
from tests import set_transformer_oracle as STO
from tests.set_transformer_oracle import STConfig, STResult, _heads, _ln_bwd, _ln_fwd, _unheads, unflatten  # noqa: F401


def mask_of(sizes, L):
    """[B, L] float64: 1 on the real particles p < l_s."""
    return (np.arange(L)[None, :] < np.asarray(sizes)[:, None]).astype(np.float64)


def forward(cfg: STConfig, flat, x, eps, sizes, beta=0.0, y=None, loss=O.LOSS_BCE_LOGITS, keep=False):
    """x [B, L, d], eps [B, L, E], sizes [B] -> prediction [B, out] (and the loss with y)."""
    p = np.asarray(flat, dtype=np.float64)
    x, eps = np.asarray(x, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    B, L, d = x.shape
    M = mask_of(sizes, L)
    ln = M.sum(1)
    Mr = M.reshape(B * L, 1)
    E, h, dk = cfg.bottleneck_dimension, cfg.number_heads, cfg.key_dim
    enc, blocks, head = unflatten(cfg, p)
    xz = np.where(M[..., None] > 0, x, 0.0)                   # padding rows enter as zeros (NaN included)
    o, acts, pres, _ = O.encoder_forward(cfg.encoder_cfg(), enc, xz.reshape(B * L, d), keep=True)
    mu, lv = o[:, :E], o[:, E:] + cfg.logvar_initialization
    u = (mu + np.exp(lv / 2.0) * np.where(Mr > 0, eps.reshape(B * L, E), 0.0)) * Mr
    kl = float((Mr * 0.5 * (mu ** 2 + np.exp(lv) - lv - 1.0)).sum() / B)
    X = u.reshape(B, L, E)
    kmask = M[:, None, None, :] > 0                           # [B, 1, 1, L] keys
    qmask = M[:, None, :, None]                               # [B, 1, L, 1] queries
    bc = []
    scale = 1.0 / math.sqrt(dk)
    for b in blocks:
        Q = _heads(X @ b["q"][0] + b["q"][1], h, dk) * scale
        K = _heads(X @ b["k"][0] + b["k"][1], h, dk)
        V = _heads(X @ b["v"][0] + b["v"][1], h, dk)
        S = np.where(kmask, Q @ K.transpose(0, 1, 3, 2), -np.inf)
        P = np.exp(S - S.max(-1, keepdims=True))
        P = P / P.sum(-1, keepdims=True) * qmask              # padding queries: zero output
        Oa = _unheads(P @ V)
        A = Oa @ b["o"][0] + b["o"][1]
        H, c1 = _ln_fwd(X + A, *b["ln1"], cfg.layer_norm_epsilon)
        F, fa = H, [H]
        for W, bb in b["ff"]:
            F = O.act_fwd(cfg.ff_activation_fn, F @ W + bb, cfg.leaky_alpha)
            fa.append(F)
        Xn, c2 = _ln_fwd(H + F, *b["ln2"], cfg.layer_norm_epsilon)
        bc.append(dict(X=X, Q=Q, K=K, V=V, P=P, O=Oa, c1=c1, fa=fa, c2=c2))
        X = Xn
    g = (X * M[..., None]).sum(1) / ln[:, None]
    ha = [g]
    for k, (W, bb) in enumerate(head):
        z = g @ W + bb
        g = O.act_fwd(cfg.activation_fn, z, cfg.leaky_alpha) if k < len(head) - 1 else z
        ha.append(g)
    res = STResult(pred=g, kl=kl, task_loss=float("nan"), loss=float("nan"), acc_sum=float("nan"))
    if y is not None and loss != "external":
        res.task_loss = float(O.task_loss_per_sample(loss, g, np.asarray(y, dtype=np.float64)).mean())
        res.loss = res.task_loss + float(beta) * kl
        res.acc_sum = O.accuracy_count(loss, g, np.asarray(y, dtype=np.float64))
    if keep:
        res.cache = dict(enc=enc, acts=acts, pres=pres, mu=mu, lv=lv, blocks=blocks, bc=bc, head=head, ha=ha, B=B, L=L, M=M,
                         eps=eps)
    return res


def train_grads(cfg: STConfig, flat, x, y, eps, sizes, beta, loss=O.LOSS_BCE_LOGITS, batch_for_mean=None):
    """Reverse mode of forward(): d(mean task loss + beta * KL)/d params, means over ``batch_for_mean`` sets (default B)."""
    fr = forward(cfg, flat, x, eps, sizes, beta, y=y, loss=loss, keep=True)
    c = fr.cache
    B, L, M = c["B"], c["L"], c["M"]
    Bm = B if batch_for_mean is None else batch_for_mean
    E, h, dk = cfg.bottleneck_dimension, cfg.number_heads, cfg.key_dim
    scale = 1.0 / math.sqrt(dk)
    y = np.asarray(y, dtype=np.float64)
    dz = y.reshape(fr.pred.shape) if loss == "external" else O.task_loss_grad(loss, fr.pred, y) / Bm
    head, ha = c["head"], c["ha"]
    hg = [None] * len(head)
    for k in reversed(range(len(head))):
        W, _ = head[k]
        hg[k] = (ha[k].T @ dz, dz.sum(0))
        dh = dz @ W.T
        if k > 0:
            dz = dh * O.act_grad_from_output(cfg.activation_fn, ha[k], cfg.leaky_alpha)
    dX = dh[:, None, :] * (M / M.sum(1, keepdims=True))[..., None]
    flatr = lambda t: t.reshape(-1, t.shape[-1])
    bgs = [None] * len(c["blocks"])
    for bi in reversed(range(len(c["blocks"]))):
        b, k = c["blocks"][bi], c["bc"][bi]
        dZ2, dg2, db2 = _ln_bwd(dX, b["ln2"][0], k["c2"])
        fa = k["fa"]
        dz = dZ2 * O.act_grad_from_output(cfg.ff_activation_fn, fa[-1], cfg.leaky_alpha)
        ffg = [None] * len(b["ff"])
        for j in reversed(range(len(b["ff"]))):
            W, _ = b["ff"][j]
            ffg[j] = (flatr(fa[j]).T @ flatr(dz), flatr(dz).sum(0))
            dh = dz @ W.T
            if j > 0:
                dz = dh * O.act_grad_from_output(cfg.ff_activation_fn, fa[j], cfg.leaky_alpha)
        dZ1, dg1, db1 = _ln_bwd(dZ2 + dh, b["ln1"][0], k["c1"])
        gWo, gbo = flatr(k["O"]).T @ flatr(dZ1), flatr(dZ1).sum(0)
        dO = _heads(dZ1 @ b["o"][0].T, h, dk)
        P, Q, K, V = k["P"], k["Q"], k["K"], k["V"]
        dV = P.transpose(0, 1, 3, 2) @ dO
        dP = dO @ V.transpose(0, 1, 3, 2)
        dS = P * (dP - (dP * P).sum(-1, keepdims=True))
        dQ = (dS @ K) * scale
        dK = dS.transpose(0, 1, 3, 2) @ Q
        dq, dk_, dv = _unheads(dQ), _unheads(dK), _unheads(dV)
        Xf = flatr(k["X"])
        g = {}
        for name, dd in (("q", dq), ("k", dk_), ("v", dv)):
            g[name] = (Xf.T @ flatr(dd), flatr(dd).sum(0))
        dX = dZ1 + dq @ b["q"][0].T + dk_ @ b["k"][0].T + dv @ b["v"][0].T
        bgs[bi] = [g["q"], g["k"], g["v"], (gWo, gbo), (dg1, db1)] + ffg + [(dg2, db2)]
    Mr = M.reshape(B * L, 1)
    du = dX.reshape(B * L, E)
    mu, lv = c["mu"], c["lv"]
    eps = np.where(Mr > 0, c["eps"].reshape(B * L, E), 0.0)
    dmu = (du + beta * mu / Bm) * Mr
    dlv = (du * eps * 0.5 * np.exp(lv / 2.0) + beta * 0.5 * (np.exp(lv) - 1.0) / Bm) * Mr
    dz = np.concatenate([dmu, dlv], -1)
    enc, acts, pres = c["enc"], c["acts"], c["pres"]
    eg = [None] * len(enc)
    for k in reversed(range(len(enc))):
        W, _ = enc[k]
        eg[k] = (acts[k].T @ dz, dz.sum(0))
        if k > 0:
            dz = (dz @ W.T) * O.act_grad_from_output(cfg.activation_fn, pres[k], cfg.leaky_alpha)
    out = [a.ravel() for pair in eg for a in pair]
    for bg in bgs:
        out += [a.ravel() for pair in bg for a in pair]
    out += [a.ravel() for pair in hg for a in pair]
    return np.concatenate(out), fr


def torch_loss(cfg: STConfig, flat, x, y, eps, sizes, beta, batch_for_mean=None):
    """The masked forward in torch float64 for autograd: (mean BCE-on-logits + beta * KL over batch_for_mean sets, flat leaf)."""
    p = torch.tensor(np.asarray(flat, dtype=np.float64), requires_grad=True)
    x, eps = torch.as_tensor(np.asarray(x, np.float64)), torch.as_tensor(np.asarray(eps, np.float64))
    y = torch.as_tensor(np.asarray(y, np.float64))
    B, L, d = x.shape
    M = torch.as_tensor(mask_of(sizes, L))
    Mr = M.reshape(B * L, 1)
    Bm = B if batch_for_mean is None else batch_for_mean
    E, h, dk = cfg.bottleneck_dimension, cfg.number_heads, cfg.key_dim
    views, off = [], 0
    for s in cfg.param_shapes():
        n = int(np.prod(s))
        views.append(p[off:off + n].reshape(s))
        off += n
    it = iter(views)
    act = lambda name, z: {"relu": torch.relu, "leaky_relu": lambda t: torch.where(t > 0, t, cfg.leaky_alpha * t),
                           "tanh": torch.tanh, None: lambda t: t, "linear": lambda t: t}[name](z)
    n = cfg.number_positional_encoding_frequencies
    hcur = torch.where(Mr > 0, x.reshape(B * L, d), 0.0)
    if n > 1:
        hcur = torch.cat([hcur] + [torch.sin(2 ** k * hcur) for k in range(1, n)], -1)
    nl = len(cfg.particle_encoder_arch_spec) + 1
    for k in range(nl):
        W, b = next(it), next(it)
        hcur = hcur @ W + b
        if k < nl - 1:
            hcur = act(cfg.activation_fn, hcur)
    mu, lv = hcur[:, :E], hcur[:, E:] + cfg.logvar_initialization
    u = (mu + torch.exp(lv / 2) * torch.where(Mr > 0, eps.reshape(B * L, E), 0.0)) * Mr
    kl = (Mr * 0.5 * (mu ** 2 + torch.exp(lv) - lv - 1)).sum() / Bm
    X = u.reshape(B, L, E)

    def ln(z, g, b):
        m = z.mean(-1, keepdim=True)
        v = ((z - m) ** 2).mean(-1, keepdim=True)
        return (z - m) / torch.sqrt(v + cfg.layer_norm_epsilon) * g + b

    kmask = M[:, None, None, :] > 0
    for _ in range(cfg.number_attention_blocks):
        Wq, bq, Wk, bk, Wv, bv, Wo, bo, g1, b1 = [next(it) for _ in range(10)]
        sh = lambda t: t.reshape(B, L, h, dk).transpose(1, 2)
        Q, K, V = sh(X @ Wq + bq) / math.sqrt(dk), sh(X @ Wk + bk), sh(X @ Wv + bv)
        Pm = torch.softmax((Q @ K.transpose(-1, -2)).masked_fill(~kmask, float("-inf")), -1) * M[:, None, :, None]
        A = (Pm @ V).transpose(1, 2).reshape(B, L, h * dk) @ Wo + bo
        H = ln(X + A, g1, b1)
        F = H
        for _ in cfg.ff_arch_per_block:
            W, b = next(it), next(it)
            F = act(cfg.ff_activation_fn, F @ W + b)
        g2, b2 = next(it), next(it)
        X = ln(H + F, g2, b2)
    g = (X * M[..., None]).sum(1) / M.sum(1, keepdim=True)
    nh = len(cfg.final_processing_arch) + 1
    for k in range(nh):
        W, b = next(it), next(it)
        g = g @ W + b
        if k < nh - 1:
            g = act(cfg.activation_fn, g)
    z, t = g, y.reshape(g.shape)
    bce = (torch.clamp(z, min=0) - z * t + torch.log1p(torch.exp(-torch.abs(z)))).mean(-1).sum() / Bm
    return bce + beta * kl, p


def fit(cfg: STConfig, flat, x, y, sizes, *, epochs, batch_size, lr, eps_fn, perm_fn, beta_fn, validation_data=None,
        loss=O.LOSS_BCE_LOGITS):
    """STO.fit on padded ragged sets: the sizes are permuted with their sets.  validation_data = (x, y, sizes)."""
    p = np.array(flat, dtype=np.float64, copy=True)
    st = O.AdamState(np.zeros_like(p), np.zeros_like(p))
    N = x.shape[0]
    sizes = np.asarray(sizes)
    keys = ["loss", "accuracy", "beta", "KL0"]
    hist = {k: [] for k in keys + (["val_" + k for k in keys] if validation_data is not None else [])}
    step = 0
    for epoch in range(epochs):
        beta = float(beta_fn(epoch))
        perm = perm_fn(epoch, N)
        s = dict(loss=0.0, acc=0.0, n=0, kl=0.0, nb=0)
        for b0 in range(0, N, batch_size):
            idx = perm[b0:b0 + batch_size]
            g, fr = train_grads(cfg, p, x[idx], y[idx], eps_fn(step, np.arange(len(idx))), sizes[idx], beta, loss)
            O.adam_step(p, g, st, lr)
            s["loss"] += fr.loss * len(idx); s["acc"] += fr.acc_sum; s["n"] += len(idx); s["kl"] += fr.kl; s["nb"] += 1
            step += 1
        hist["loss"].append(s["loss"] / s["n"]); hist["accuracy"].append(s["acc"] / s["n"])
        hist["beta"].append(beta); hist["KL0"].append(s["kl"] / s["nb"])
        if validation_data is not None:
            xv, yv, sv = validation_data
            v = dict(loss=0.0, acc=0.0, n=0, kl=0.0, nb=0)
            for b0 in range(0, xv.shape[0], batch_size):
                idx = np.arange(b0, min(b0 + batch_size, xv.shape[0]))
                fr = forward(cfg, p, xv[idx], eps_fn(2 ** 31 + epoch, idx), np.asarray(sv)[idx], beta, y=yv[idx], loss=loss)
                v["loss"] += fr.loss * len(idx); v["acc"] += fr.acc_sum; v["n"] += len(idx); v["kl"] += fr.kl; v["nb"] += 1
            hist["val_loss"].append(v["loss"] / v["n"]); hist["val_accuracy"].append(v["acc"] / v["n"])
            hist["val_beta"].append(beta); hist["val_KL0"].append(v["kl"] / v["nb"])
    return p, hist


__all__ = ["forward", "train_grads", "torch_loss", "fit", "mask_of", "STO"]
