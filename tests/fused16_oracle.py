"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the 16-bit fused training path ('fp16' / 'bf16' precision) that rounds
to 16 bits exactly where the kernels round.  Not collected by pytest (no test_ prefix).

The fused path is deterministic and its arithmetic explicit: every activation and gradient operand is rounded to 16 bits
(`cvt.rn.satfinite`) at a known point, the weights once when they are packed, every MMA accumulates in fp32, and the loss
scale S is a power of two.  Everything here is float64 except those roundings, which are applied to the float64 value
directly, so the kernels should differ from this oracle only by fp32 accumulation, the SFU approximations (`__sinf`,
`__expf`, `tanh.approx`) and the one-ulp rounding flips those cause.  With ``fmt=None`` no rounding happens and the functions
equal oracle/dib_oracle.py's ``forward`` / ``train_grads``: the two oracles differ only in the rounding points listed below.

Rounding points (kernel files under distributed-information-bottleneck.github.io_b200/csrc/):
  encoder forward (dib_enc_fused.cu)
    * [pe | 1] operand                          write_a0_row :214-235 (pack2 of the sin / x values)
    * W0, W1, W2, b0, b1, b2 + logvar_offset    dib_enc_pack_weights_kernel :733-765 (biases enter as bias-carrier rows)
    * h1 = r(act(z1)), h2 = r(act(z2))          frag_to_a :152 (forward), frag_to_tile :137 (recomputed in the backward)
    * (mu, logvar) = the fp32 accumulator; u = mu + exp(logvar / 2) eps and KL in fp32 (:460-469)
    * emb16 = r(u); the user-visible emb is u itself (:470-471)
  integration network (dib_int16.cu)
    * W_j of the hidden layers                  dib_f32_to_16_segs_kernel :959 (biases, head weights and bias stay fp32)
    * g_{j+1} = r(act(g_j W_j + b_j))           FWD epilogue :215, fused tail e0 :443 and e1 :462
    * logit = g_L . w + b in fp32               e1 :470, head kernels :667 / :808
    * dzs = dloss * inv_batch * out_act'(z), ds = dzs * S     :491-492, :701, :838
    * dg_{L-1} = r(ds w act'(g_L)); its column sums (bias gradient) are of the unrounded values   :507-510, :708-709, :849-850
    * dg_j = r((dg_{j+1} W_{j+1}^T) act'(g_{j+1})), bias gradient from unrounded values          DGRAD :220-224, e2 :548-554
    * d_emb16 = r(dg_0 W_0^T)                   DGRAD without act' (g_in = null), fused tail e3 :582
    * output layer: dW = g_L^T dzs, db = sum dzs (no S); hidden dW_j = g_j^T dg_j / S (WGRAD :212); bias sums / S (dib_api.cu:926, :942)
  encoder backward (dib_enc_fused.cu)
    * g = d_emb16 as stored, or the fp32 d_emb times S (:619-622); bs = beta_eff * inv_batch * S (:567)
    * dO = r([g + bs mu | g eps sigma / 2 + bs (sigma^2 - 1) / 2])   :627-634
    * dz2 = r(G2 act'(h2)), dz1 = r(G1 act'(h1))   frag_dgrad_to_tile :180-199 (relu: rounded, then gated -- the same value)
    * dW2 = h2^T dO, dW1 = h1^T dz2, [dW0; db0] = dz1^T [pe | 1]; db2 / db1 are column sums of the 16-bit dO / dz2 (the ones
      column of [pe | 1] is an MMA operand); everything * 1/S on the flush (:696)
"""
from __future__ import annotations

import math

import numpy as np

from oracle import dib_oracle as O

# significand bits t (incl. the implicit one), minimum normal exponent, largest finite value
FORMATS = {
    "fp16": (11, -14, 65504.0),
    "bf16": (8, -126, (2.0 - 2.0 ** -7) * 2.0 ** 127),
}


def round_to(x, fmt, saturate=True):
    """Round half to even to the 16-bit format ``fmt`` ('fp16' | 'bf16' | None = no rounding), in float64.  Subnormals are
    exact (the quantum never drops below 2^(emin - t + 1)).  ``saturate``: a result beyond the largest finite value becomes
    +-max (cvt.rn.satfinite; infinities too), else +-inf (cvt.rn / __float2half_rn).  NaN stays NaN."""
    x = np.asarray(x, dtype=np.float64)
    if fmt is None:
        return x
    t, emin, vmax = FORMATS[fmt]
    finite = np.isfinite(x)
    xf = np.where(finite, x, 0.0)
    _, ex = np.frexp(xf)                                    # |x| = m 2^ex, m in [0.5, 1): leading bit 2^(ex - 1)
    e = np.maximum(ex - 1, emin)
    q = np.ldexp(1.0, e - (t - 1))                          # the quantum (ulp) at that exponent
    r = np.round(xf / q) * q                                # x / q is exact (power-of-two scaling); np.round: half to even
    if saturate:
        r = np.clip(r, -vmax, vmax)
        r = np.where(np.isinf(x), np.sign(x) * vmax, r)
    else:
        r = np.where(np.abs(r) > vmax, np.copysign(np.inf, r), r)
        r = np.where(np.isinf(x), x, r)
    return np.where(np.isnan(x), np.nan, r)


def loss_scale(global_batch):
    """S = 2^ceil(log2 B_global) (dib_api.cu:174)."""
    return float(2.0 ** math.ceil(math.log2(max(int(global_batch), 1))))


def _act(cfg, z):
    return O.act_fwd(cfg.activation_fn, z, cfg.leaky_alpha)


def _dact(cfg, h):
    return O.act_grad_from_output(cfg.activation_fn, h, cfg.leaky_alpha)


def _encoder_forward(cfg, layers, x_i, fmt):
    """One feature encoder in the fused kernel's arithmetic: returns (a0 = r(pe), h1, h2, mu, logvar)."""
    assert cfg.encoder_kind == "mlp" and len(layers) == 3, "the fused encoder kernels run [hidden, hidden, 2E] encoders"
    R = lambda v: round_to(v, fmt)
    E = cfg.feature_embedding_dimension
    (W0, b0), (W1, b1), (W2, b2) = layers
    pe = O.positional_encoding(x_i, cfg.frequencies) if cfg.use_positional_encoding else x_i
    a0 = R(pe)                                                          # write_a0_row :234
    h1 = R(_act(cfg, a0 @ R(W0) + R(b0)))                               # pack :749 (b0 = row w_in of W0p); frag_to_a :436
    h2 = R(_act(cfg, R(b1) + h1 @ R(W1)))                               # bias-carrier step first (:351), then W1; :442
    off = np.concatenate([np.zeros(E), np.full(E, cfg.logvar_offset)])
    o = R(b2 + off) + h2 @ R(W2)                                        # pack :760: the offset is inside the rounded carrier
    return a0, h1, h2, o[:, :E], o[:, E:]


def forward(cfg, flat, x, eps, beta, y=None, loss=None, fmt=None, keep=False):
    """The training / inference forward of the fused path.  Returns an O.ForwardResult whose ``emb`` is the unrounded u (what
    the kernel hands back as the fp32 embedding) and whose cache also holds ``emb16`` = r(u) and the per-layer 16-bit values."""
    p = np.asarray(flat, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    eps = np.asarray(eps, dtype=np.float64)
    encoders, integration = O.unflatten(cfg, p)
    xs = O.split_features(cfg, x)
    R = lambda v: round_to(v, fmt)
    enc, embs, kls = [], [], []
    for i in range(cfg.number_features):
        a0, h1, h2, mu, lv = _encoder_forward(cfg, encoders[i], xs[i], fmt)
        sig = np.exp(lv / 2.0)
        embs.append(mu + sig * eps[:, i, :])                            # :466-467
        kls.append((0.5 * (mu ** 2 + (np.expm1(lv) - lv))).sum(axis=-1).mean())   # :493 (sv * sv - lv - 1)
        enc.append((a0, h1, h2, mu, lv))
    emb = np.concatenate(embs, axis=-1)
    g = R(emb)                                                          # emb16 :471
    acts = [g]
    for j, (W, b) in enumerate(integration[:-1]):
        g = R(_act(cfg, g @ R(W) + b))                                  # FWD :215, e0 :443, e1 :462 (bias fp32)
        acts.append(g)
    Wc, bc = integration[-1]
    pred = O.act_fwd(cfg.output_activation_fn, g @ Wc + bc, cfg.leaky_alpha)   # head weights stay fp32
    kls = np.asarray(kls)
    res = O.ForwardResult(pred=pred, emb=emb, kl_per_feature=kls, task_loss=float("nan"), loss=float("nan"),
                          acc_sum=float("nan"))
    if y is not None:
        per = O.task_loss_per_sample(loss, pred, y)
        res.task_loss = float(per.mean())
        res.loss = res.task_loss + O.ib_loss(cfg, beta, kls)
        res.acc_sum = O.accuracy_count(loss, pred, y)
        res.cache["loss_sum"] = float(per.sum())
    res.cache.update(enc=enc, int_acts=acts, encoders=encoders, integration=integration, emb16=acts[0])
    return res


def encoder_backward(cfg, fr, eps, g_emb, beta_eff, B, S, fmt):
    """The fused encoder backward (dib_enc_fused_bwd_kernel) from ``g_emb`` = the S-scaled gradient w.r.t. emb (d_emb16 as
    stored, or the fp32 d_emb times S).  Returns the flat encoder gradients [per feature: W0, b0, W1, b1, W2, b2]."""
    R = lambda v: round_to(v, fmt)
    E = cfg.feature_embedding_dimension
    eps = np.asarray(eps, dtype=np.float64)
    bs = beta_eff / B * S                                               # :567
    out = []
    for i in range(cfg.number_features):
        a0, h1, h2, mu, lv = fr.cache["enc"][i]
        (W0, _), (W1, _), (W2, _) = fr.cache["encoders"][i]
        g = g_emb[:, i * E:(i + 1) * E]
        sig = np.exp(lv / 2.0)
        dO = R(np.concatenate([g + bs * mu, g * eps[:, i, :] * 0.5 * sig + bs * 0.5 * (sig * sig - 1.0)], axis=-1))   # :630-634
        dz2 = R((dO @ R(W2).T) * _dact(cfg, h2))                        # frag_dgrad_to_tile :657
        dz1 = R((dz2 @ R(W1).T) * _dact(cfg, h1))                       # :678
        w_in = W0.shape[0]
        out += [(a0[:, :w_in].T @ dz1).ravel() / S, dz1.sum(axis=0) / S,                    # :686, :715-717
                (h1.T @ dz2).ravel() / S, dz2.sum(axis=0) / S,                              # :670-673
                (h2.T @ dO).ravel() / S, dO.sum(axis=0) / S]                                # :648-652
    return np.concatenate(out)


def train_grads(cfg, flat, x, y, eps, beta, loss, fmt=None, S=None, batch_for_mean=None, d_emb=None):
    """Signature of O.train_grads plus ``fmt`` and the loss scale ``S`` (default 2^ceil(log2 B_global)).  ``d_emb`` given:
    the encoder-only step of ``encoder_gradients`` (fp32 d_emb, already carrying the caller's 1/B; integration entries 0).
    Returns (flat grads, ForwardResult); the result's cache holds ``d_emb16`` (the S-scaled 16-bit embedding gradient)."""
    fr = forward(cfg, flat, x, eps, beta, y=None if d_emb is not None else y, loss=loss, fmt=fmt)
    n = x.shape[0]
    B = n if batch_for_mean is None else batch_for_mean
    S = loss_scale(B) if S is None else float(S)
    R = lambda v: round_to(v, fmt)
    beta_eff = O.effective_beta(cfg, beta, fr.kl_per_feature * (n / B))
    integration, acts = fr.cache["integration"], fr.cache["int_acts"]
    Li = len(integration) - 1
    if d_emb is not None:
        g_emb = np.asarray(d_emb, dtype=np.float64).reshape(fr.emb.shape) * S            # :622
        int_grads = [np.zeros(W.size + b.size) for W, b in integration]
    else:
        Wc, _ = integration[-1]
        dzs = O.task_loss_grad(loss, fr.pred, y) / B * O.act_grad_from_output(cfg.output_activation_fn, fr.pred, cfg.leaky_alpha)
        int_grads = [None] * (Li + 1)
        int_grads[Li] = np.concatenate([(acts[Li].T @ dzs).ravel(), dzs.sum(axis=0)])     # :508 / :707 (no S)
        d = (S * dzs) @ Wc.T * _dact(cfg, acts[Li])                                        # :507 / :708 / :849
        for j in range(Li - 1, -1, -1):
            dg = R(d)
            W, _ = integration[j]
            int_grads[j] = np.concatenate([(acts[j].T @ dg).ravel() / S, d.sum(axis=0) / S])   # WGRAD :212; bias sums
            d = dg @ R(W).T
            if j > 0:
                d = d * _dact(cfg, acts[j])                                                # DGRAD :220, e2 :548
        g_emb = R(d)                                                                       # d_emb16: e3 :582 / DGRAD
        fr.cache["d_emb16"] = g_emb
    enc = encoder_backward(cfg, fr, eps, g_emb, beta_eff, B, S, fmt)
    return np.concatenate([enc] + [g.ravel() for g in int_grads]), fr


def per_variable_errors(cfg, g, g_ref):
    """max |g - g_ref| / max |g_ref| of every variable of the flat layout (0 where the reference is all zero and g equals it)."""
    out, off = [], 0
    for s in cfg.param_shapes():
        k = int(np.prod(s))
        a, b = np.asarray(g[off:off + k], np.float64), np.asarray(g_ref[off:off + k], np.float64)
        den = np.abs(b).max()
        out.append(float(np.abs(a - b).max() / den) if den > 0 else float(np.abs(a).max()))
        off += k
    return np.asarray(out)
