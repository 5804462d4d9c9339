"""TEST INFRASTRUCTURE ONLY -- float64 restatement of nb-particle cell 8's per-particle set transformer (BASELINE config 5):
the shared particle encoder (oracle/dib_oracle.py's encoder on particle rows), ``number_attention_blocks`` blocks of
Keras 2 MultiHeadAttention (no dropout, no mask) + LayerNorm + FF + LayerNorm, the mean over the particles and the Dense head.
A hand-written reverse mode, a PyTorch float64 autograd twin to check it against, and a Model.fit-style epoch loop.  The
product path never imports this module."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import torch

from oracle import dib_oracle as O


@dataclass
class STConfig:
    particle_feature_dimensions: int = 12
    particle_encoder_arch_spec: Sequence[int] = (128, 128)
    bottleneck_dimension: int = 32
    number_particles: int = 50
    key_dim: int = 128
    number_heads: int = 12
    number_attention_blocks: int = 6
    ff_arch_per_block: Sequence[int] = field(default_factory=lambda: [128, 32])
    ff_activation_fn: str = "relu"
    final_processing_arch: Sequence[int] = (256,)
    activation_fn: str = "leaky_relu"
    leaky_alpha: float = 0.1
    output_dimensionality: int = 1
    logvar_initialization: float = -3.0
    number_positional_encoding_frequencies: int = 5
    layer_norm_epsilon: float = 1e-3            # [KERAS] LayerNormalization default

    def encoder_cfg(self):
        """The particle encoder as a one-feature DIBConfig (its integration layers are not used)."""
        n = self.number_positional_encoding_frequencies
        return O.DIBConfig([self.particle_feature_dimensions], list(self.particle_encoder_arch_spec), [], 1,
                           use_positional_encoding=n > 1, number_positional_encoding_frequencies=n,
                           activation_fn=self.activation_fn, feature_embedding_dimension=self.bottleneck_dimension,
                           leaky_alpha=self.leaky_alpha, logvar_offset=self.logvar_initialization)

    def param_shapes(self):
        """Flat order (all_trainable_variables): encoder Dense (W, b)..., per block q W [E, h*dk], q b, k, k b, v, v b,
        output W [h*dk, E], output b, LN1 gamma, beta, FF (W, b)..., LN2 gamma, beta; then the head's Dense (W, b)..."""
        E, hd = self.bottleneck_dimension, self.number_heads * self.key_dim
        d = self.encoder_cfg().encoder_layer_dims(0)
        shapes = []
        for k in range(len(d) - 1):
            shapes += [(d[k], d[k + 1]), (d[k + 1],)]
        ff = [E] + list(self.ff_arch_per_block)
        for _ in range(self.number_attention_blocks):
            shapes += [(E, hd), (hd,)] * 3 + [(hd, E), (E,), (E,), (E,)]
            for k in range(len(ff) - 1):
                shapes += [(ff[k], ff[k + 1]), (ff[k + 1],)]
            shapes += [(E,), (E,)]
        hd_ = [E] + list(self.final_processing_arch) + [self.output_dimensionality]
        for k in range(len(hd_) - 1):
            shapes += [(hd_[k], hd_[k + 1]), (hd_[k + 1],)]
        return shapes

    def param_count(self):
        return int(sum(int(np.prod(s)) for s in self.param_shapes()))

    def encoder_param_count(self):
        d = self.encoder_cfg().encoder_layer_dims(0)
        return int(sum(d[k] * d[k + 1] + d[k + 1] for k in range(len(d) - 1)))


def init_params(cfg: STConfig, rng: np.random.Generator, dtype=np.float32):
    """[KERAS] glorot_uniform kernels (the 3-D attention kernels with _compute_fans' fans), zero biases, LayerNorm gamma = 1,
    then small random biases / LayerNorm offsets so that every parameter is exercised (our RNG stream)."""
    E, h, dk = cfg.bottleneck_dimension, cfg.number_heads, cfg.key_dim
    out = []
    shapes = cfg.param_shapes()
    n_enc = 2 * (len(cfg.particle_encoder_arch_spec) + 1)
    per_block = 12 + 2 * len(cfg.ff_arch_per_block)
    for i, s in enumerate(shapes):
        j = (i - n_enc) % per_block if n_enc <= i < n_enc + per_block * cfg.number_attention_blocks else -1
        if len(s) == 2:
            if j in (0, 2, 4):
                fi, fo = h * E, dk * E
            elif j == 6:
                fi, fo = dk * h, E * h
            else:
                fi, fo = s
            lim = math.sqrt(6.0 / (fi + fo))
            out.append(rng.uniform(-lim, lim, size=s).ravel())
        elif j in (8, per_block - 2):                       # LayerNorm gamma
            out.append(1.0 + 0.1 * rng.standard_normal(s))
        else:
            out.append(0.05 * rng.standard_normal(s))
    return np.concatenate(out).astype(dtype)


def unflatten(cfg: STConfig, flat):
    views, off = [], 0
    for s in cfg.param_shapes():
        n = int(np.prod(s))
        views.append(flat[off:off + n].reshape(s))
        off += n
    assert off == flat.size, (off, flat.size)
    it = iter(views)
    enc = [(next(it), next(it)) for _ in range(len(cfg.particle_encoder_arch_spec) + 1)]
    blocks = []
    for _ in range(cfg.number_attention_blocks):
        b = dict(q=(next(it), next(it)), k=(next(it), next(it)), v=(next(it), next(it)), o=(next(it), next(it)),
                 ln1=(next(it), next(it)))
        b["ff"] = [(next(it), next(it)) for _ in cfg.ff_arch_per_block]
        b["ln2"] = (next(it), next(it))
        blocks.append(b)
    head = [(next(it), next(it)) for _ in range(len(cfg.final_processing_arch) + 1)]
    return enc, blocks, head


def _ln_fwd(z, gamma, beta, eps):
    mean = z.mean(-1, keepdims=True)
    var = ((z - mean) ** 2).mean(-1, keepdims=True)           # biased variance
    rstd = 1.0 / np.sqrt(var + eps)
    xhat = (z - mean) * rstd
    return xhat * gamma + beta, (xhat, rstd)


def _ln_bwd(dy, gamma, cache):
    xhat, rstd = cache
    g = dy * gamma
    dz = rstd * (g - g.mean(-1, keepdims=True) - xhat * (g * xhat).mean(-1, keepdims=True))
    return dz, (dy * xhat).reshape(-1, xhat.shape[-1]).sum(0), dy.reshape(-1, xhat.shape[-1]).sum(0)


def _heads(t, h, dk):           # [B, L, h*dk] -> [B, h, L, dk]
    B, L = t.shape[:2]
    return t.reshape(B, L, h, dk).transpose(0, 2, 1, 3)


def _unheads(t):                # [B, h, L, dk] -> [B, L, h*dk]
    B, h, L, dk = t.shape
    return t.transpose(0, 2, 1, 3).reshape(B, L, h * dk)


@dataclass
class STResult:
    pred: np.ndarray
    kl: float                   # sum over particles and dims, mean over sets
    task_loss: float
    loss: float
    acc_sum: float
    cache: dict = field(default_factory=dict)


def forward(cfg: STConfig, flat, x, eps, beta=0.0, y=None, loss=O.LOSS_BCE_LOGITS, keep=False):
    """x [B, L, d], eps [B, L, E] -> prediction [B, out] (and the loss with y)."""
    p = np.asarray(flat, dtype=np.float64)
    x, eps = np.asarray(x, dtype=np.float64), np.asarray(eps, dtype=np.float64)
    B, L, d = x.shape
    E, h, dk = cfg.bottleneck_dimension, cfg.number_heads, cfg.key_dim
    enc, blocks, head = unflatten(cfg, p)
    ecfg = cfg.encoder_cfg()
    o, acts, pres, _ = O.encoder_forward(ecfg, enc, x.reshape(B * L, d), keep=True)
    mu, lv = o[:, :E], o[:, E:] + cfg.logvar_initialization
    u = mu + np.exp(lv / 2.0) * eps.reshape(B * L, E)
    kl = float((0.5 * (mu ** 2 + np.exp(lv) - lv - 1.0)).sum() / B)
    X = u.reshape(B, L, E)
    bc = []
    scale = 1.0 / math.sqrt(dk)
    for b in blocks:
        Q = _heads(X @ b["q"][0] + b["q"][1], h, dk) * scale
        K = _heads(X @ b["k"][0] + b["k"][1], h, dk)
        V = _heads(X @ b["v"][0] + b["v"][1], h, dk)
        S = Q @ K.transpose(0, 1, 3, 2)
        P = np.exp(S - S.max(-1, keepdims=True))
        P /= P.sum(-1, keepdims=True)
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
    g = X.mean(1)
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
        res.cache = dict(enc=enc, acts=acts, pres=pres, mu=mu, lv=lv, blocks=blocks, bc=bc, head=head, ha=ha, B=B, L=L)
    return res


def train_grads(cfg: STConfig, flat, x, y, eps, beta, loss=O.LOSS_BCE_LOGITS, batch_for_mean=None):
    """Reverse mode of forward(): d(mean task loss + beta * KL)/d params, means over ``batch_for_mean`` sets (default B)."""
    fr = forward(cfg, flat, x, eps, beta, y=y, loss=loss, keep=True)
    c = fr.cache
    B, L = c["B"], c["L"]
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
    dX = np.repeat(dh[:, None, :] / L, L, axis=1)
    bgs = [None] * len(c["blocks"])
    for bi in reversed(range(len(c["blocks"]))):
        b, k = c["blocks"][bi], c["bc"][bi]
        dZ2, dg2, db2 = _ln_bwd(dX, b["ln2"][0], k["c2"])
        fa = k["fa"]
        dz = dZ2 * O.act_grad_from_output(cfg.ff_activation_fn, fa[-1], cfg.leaky_alpha)
        ffg = [None] * len(b["ff"])
        for j in reversed(range(len(b["ff"]))):
            W, _ = b["ff"][j]
            ffg[j] = (fa[j].reshape(-1, fa[j].shape[-1]).T @ dz.reshape(-1, dz.shape[-1]), dz.reshape(-1, dz.shape[-1]).sum(0))
            dh = dz @ W.T
            if j > 0:
                dz = dh * O.act_grad_from_output(cfg.ff_activation_fn, fa[j], cfg.leaky_alpha)
        dZ1, dg1, db1 = _ln_bwd(dZ2 + dh, b["ln1"][0], k["c1"])
        flatr = lambda t: t.reshape(-1, t.shape[-1])
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
    # encoder: d u, plus beta * dKL / Bm per particle row
    du = dX.reshape(B * L, E)
    mu, lv = c["mu"], c["lv"]
    eps = np.asarray(eps, dtype=np.float64).reshape(B * L, E)
    dmu = du + beta * mu / Bm
    dlv = du * eps * 0.5 * np.exp(lv / 2.0) + beta * 0.5 * (np.exp(lv) - 1.0) / Bm
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


def torch_loss(cfg: STConfig, flat, x, y, eps, beta, batch_for_mean=None):
    """The same forward in torch float64 for autograd: returns (mean BCE-on-logits + beta * KL over batch_for_mean sets,
    flat parameter leaf)."""
    p = torch.tensor(np.asarray(flat, dtype=np.float64), requires_grad=True)
    x, eps = torch.as_tensor(np.asarray(x, np.float64)), torch.as_tensor(np.asarray(eps, np.float64))
    y = torch.as_tensor(np.asarray(y, np.float64))
    B, L, d = x.shape
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
    hcur = x.reshape(B * L, d)
    if n > 1:
        hcur = torch.cat([hcur] + [torch.sin(2 ** k * hcur) for k in range(1, n)], -1)
    nl = len(cfg.particle_encoder_arch_spec) + 1
    for k in range(nl):
        W, b = next(it), next(it)
        hcur = hcur @ W + b
        if k < nl - 1:
            hcur = act(cfg.activation_fn, hcur)
    mu, lv = hcur[:, :E], hcur[:, E:] + cfg.logvar_initialization
    u = mu + torch.exp(lv / 2) * eps.reshape(B * L, E)
    kl = (0.5 * (mu ** 2 + torch.exp(lv) - lv - 1)).sum() / Bm
    X = u.reshape(B, L, E)

    def ln(z, g, b):
        m = z.mean(-1, keepdim=True)
        v = ((z - m) ** 2).mean(-1, keepdim=True)
        return (z - m) / torch.sqrt(v + cfg.layer_norm_epsilon) * g + b

    for _ in range(cfg.number_attention_blocks):
        Wq, bq, Wk, bk, Wv, bv, Wo, bo, g1, b1 = [next(it) for _ in range(10)]
        sh = lambda t: t.reshape(B, L, h, dk).transpose(1, 2)
        Q, K, V = sh(X @ Wq + bq) / math.sqrt(dk), sh(X @ Wk + bk), sh(X @ Wv + bv)
        Pm = torch.softmax(Q @ K.transpose(-1, -2), -1)
        A = (Pm @ V).transpose(1, 2).reshape(B, L, h * dk) @ Wo + bo
        H = ln(X + A, g1, b1)
        F = H
        for _ in cfg.ff_arch_per_block:
            W, b = next(it), next(it)
            F = act(cfg.ff_activation_fn, F @ W + b)
        g2, b2 = next(it), next(it)
        X = ln(H + F, g2, b2)
    g = X.mean(1)
    nh = len(cfg.final_processing_arch) + 1
    for k in range(nh):
        W, b = next(it), next(it)
        g = g @ W + b
        if k < nh - 1:
            g = act(cfg.activation_fn, g)
    z, t = g, y.reshape(g.shape)
    bce = (torch.clamp(z, min=0) - z * t + torch.log1p(torch.exp(-torch.abs(z)))).mean(-1).sum() / Bm
    return bce + beta * kl, p


def fit(cfg: STConfig, flat, x, y, *, epochs, batch_size, lr, eps_fn, perm_fn, beta_fn, validation_data=None,
        loss=O.LOSS_BCE_LOGITS):
    """Model.fit around the set transformer, as O.fit does it for DistributedIBNet: beta at epoch begin, consecutive batches
    of the epoch permutation with a short last one, Keras Adam, running means (loss and accuracy sample-weighted, KL0 and beta
    over batches) and a validation pass in batches of batch_size.  eps_fn(step, set_ids) -> eps [n, L, E]."""
    p = np.array(flat, dtype=np.float64, copy=True)
    st = O.AdamState(np.zeros_like(p), np.zeros_like(p))
    N = x.shape[0]
    keys = ["loss", "accuracy", "beta", "KL0"]
    hist = {k: [] for k in keys + (["val_" + k for k in keys] if validation_data is not None else [])}
    step = 0
    for epoch in range(epochs):
        beta = float(beta_fn(epoch))
        perm = perm_fn(epoch, N)
        s = dict(loss=0.0, acc=0.0, n=0, kl=0.0, nb=0)
        for b0 in range(0, N, batch_size):
            idx = perm[b0:b0 + batch_size]
            g, fr = train_grads(cfg, p, x[idx], y[idx], eps_fn(step, np.arange(len(idx))), beta, loss)
            O.adam_step(p, g, st, lr)
            s["loss"] += fr.loss * len(idx); s["acc"] += fr.acc_sum; s["n"] += len(idx); s["kl"] += fr.kl; s["nb"] += 1
            step += 1
        hist["loss"].append(s["loss"] / s["n"]); hist["accuracy"].append(s["acc"] / s["n"])
        hist["beta"].append(beta); hist["KL0"].append(s["kl"] / s["nb"])
        if validation_data is not None:
            xv, yv = validation_data
            v = dict(loss=0.0, acc=0.0, n=0, kl=0.0, nb=0)
            for b0 in range(0, xv.shape[0], batch_size):
                idx = np.arange(b0, min(b0 + batch_size, xv.shape[0]))
                fr = forward(cfg, p, xv[idx], eps_fn(2 ** 31 + epoch, idx), beta, y=yv[idx], loss=loss)
                v["loss"] += fr.loss * len(idx); v["acc"] += fr.acc_sum; v["n"] += len(idx); v["kl"] += fr.kl; v["nb"] += 1
            hist["val_loss"].append(v["loss"] / v["n"]); hist["val_accuracy"].append(v["acc"] / v["n"])
            hist["val_beta"].append(beta); hist["val_KL0"].append(v["kl"] / v["nb"])
    return p, hist
