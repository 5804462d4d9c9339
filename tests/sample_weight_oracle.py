"""TEST INFRASTRUCTURE ONLY -- per-sample weights of the compiled loss on top of the unmodified float64 oracles.  Not collected
by pytest (no test_ prefix).

[KERAS] reduction SUM_OVER_BATCH_SIZE: task loss = sum_i w_i l_i / B with B the (global) batch size, not sum w; d loss / d z_i is
w_i times the unweighted value; beta * KL and the accuracy are not weighted.

The weighted gradient is each oracle's own reverse mode driven by the caller-owned-loss route (loss = "external": y is
d(task loss)/d(prediction), already batch-scaled), fed w_i (d l_i / d z_i) / B.  The rounding-aware 16-bit oracle has no such
route, so its integration backward is restated here (fused16_train_grads, the body of tests/fused16_oracle.py's train_grads
with w entering dzs ahead of every 16-bit rounding, as in the kernels), and so is the epoch loop of O.fit (fit).
tests/test_sample_weights_host.py pins every function here to the unweighted oracle it extends: all-ones weights give its
results exactly.
"""
from __future__ import annotations

import numpy as np

from oracle import dib_oracle as O
from tests import fused16_oracle as Q


def _w(sample_weight):
    return np.asarray(sample_weight, dtype=np.float64).reshape(-1)


def weighted_dz(loss, pred, y, sample_weight, B):
    """d(sum_i w_i l_i / B) / d pred [n, out]."""
    return O.task_loss_grad(loss, pred, y) / B * _w(sample_weight)[:, None]


def _weigh(fr, loss, pred, y, sample_weight, ib):
    """Fill a forward result's task loss (mean of w_i l_i), total loss (+ the unweighted IB term ib), loss sum and accuracy."""
    per = O.task_loss_per_sample(loss, pred, np.asarray(y, dtype=np.float64)) * _w(sample_weight)
    fr.task_loss = float(per.mean())
    fr.loss = fr.task_loss + ib
    fr.acc_sum = O.accuracy_count(loss, pred, np.asarray(y, dtype=np.float64))
    if isinstance(getattr(fr, "cache", None), dict):
        fr.cache["loss_sum"] = float(per.sum())
    return fr


# ---------------------------------------------------------------------------------------------------------------------
# oracle/dib_oracle.py
# ---------------------------------------------------------------------------------------------------------------------
def forward(cfg, flat, x, eps, beta, y, loss, sample_weight, dtype=np.float64):
    """O.forward with the task loss weighted."""
    fr = O.forward(cfg, flat, x, eps, beta, dtype=dtype)
    return _weigh(fr, loss, fr.pred, y, sample_weight, O.ib_loss(cfg, beta, fr.kl_per_feature))


def train_grads(cfg, flat, x, y, eps, beta, loss, sample_weight, dtype=np.float64, batch_for_mean=None, dropout=None):
    """O.train_grads of the weighted loss: (flat gradient, ForwardResult with the weighted task loss)."""
    B = x.shape[0] if batch_for_mean is None else batch_for_mean
    pred = O.forward(cfg, flat, x, eps, beta, dtype=dtype, dropout=dropout).pred
    g, fr = O.train_grads(cfg, flat, x, weighted_dz(loss, pred, y, sample_weight, B), eps, beta, "external", dtype=dtype,
                          batch_for_mean=B, dropout=dropout)
    return g, _weigh(fr, loss, fr.pred, y, sample_weight, O.ib_loss(cfg, beta, fr.kl_per_feature))


def fit(cfg, flat_params, x, y, *, loss, epochs, batch_size, lr, eps_fn, perm_fn=None, beta_fn=None, validation_data=None,
        dtype=np.float64, adam_kwargs=None, sample_weight=None):
    """O.fit's epoch mechanics (see there) with the training rows' task loss weighted by ``sample_weight`` [N] (None: all 1) and
    the validation loss by the third element of ``validation_data`` = (xv, yv[, wv])."""
    p = np.array(flat_params, dtype=dtype, copy=True)
    st = O.AdamState(np.zeros_like(p), np.zeros_like(p))
    N, F = x.shape[0], cfg.number_features
    w = np.ones(N) if sample_weight is None else _w(sample_weight)
    hist = {k: [] for k in ["loss", "accuracy", "beta"] + [f"KL{i}" for i in range(F)]}
    if validation_data is not None:
        for k in list(hist):
            hist["val_" + k] = []
    step, beta = 0, 1.0
    adam_kwargs = adam_kwargs or {}

    def record(prefix, sums):
        hist[prefix + "loss"].append(sums["loss"] / sums["n"])
        hist[prefix + "accuracy"].append(sums["acc"] / sums["n"])
        hist[prefix + "beta"].append(beta)
        for i in range(F):
            hist[f"{prefix}KL{i}"].append(sums["kl"][i] / sums["nb"])

    def add(sums, fr, n):
        sums["loss"] += fr.loss * n
        sums["acc"] += fr.acc_sum
        sums["n"] += n
        sums["kl"] += fr.kl_per_feature
        sums["nb"] += 1

    for epoch in range(epochs):
        if beta_fn is not None:
            beta = float(beta_fn(epoch))
        perm = perm_fn(epoch, N) if perm_fn is not None else np.arange(N)
        sums = dict(loss=0.0, acc=0.0, n=0, kl=np.zeros(F), nb=0)
        for b0 in range(0, N, batch_size):
            idx = perm[b0:b0 + batch_size]
            g, fr = train_grads(cfg, p, x[idx], y[idx], eps_fn(step, np.arange(len(idx))), beta, loss, w[idx], dtype=dtype)
            O.adam_step(p, g.astype(dtype), st, lr, **adam_kwargs)
            add(sums, fr, len(idx))
            step += 1
        record("", sums)
        if validation_data is not None:
            xv, yv = validation_data[:2]
            wv = np.ones(xv.shape[0]) if len(validation_data) < 3 else _w(validation_data[2])
            vs = dict(loss=0.0, acc=0.0, n=0, kl=np.zeros(F), nb=0)
            for b0 in range(0, xv.shape[0], batch_size):
                idx = np.arange(b0, min(b0 + batch_size, xv.shape[0]))
                add(vs, forward(cfg, p, xv[idx], eps_fn(2 ** 31 + epoch, idx), beta, yv[idx], loss, wv[idx], dtype=dtype), len(idx))
            record("val_", vs)
    return p, hist


# ---------------------------------------------------------------------------------------------------------------------
# tests/fused16_oracle.py: the 16-bit fused path's rounding points, w_i multiplying dzs (the fp32 d loss / d logit)
# ---------------------------------------------------------------------------------------------------------------------
def fused16_train_grads(cfg, flat, x, y, eps, beta, loss, sample_weight, fmt=None, S=None, batch_for_mean=None):
    """Q.train_grads (the non-encoder-only route) of the weighted loss: (flat gradient, ForwardResult)."""
    fr = Q.forward(cfg, flat, x, eps, beta, y=y, loss=loss, fmt=fmt)
    n = x.shape[0]
    B = n if batch_for_mean is None else batch_for_mean
    S = Q.loss_scale(B) if S is None else float(S)
    R = lambda v: Q.round_to(v, fmt)
    beta_eff = O.effective_beta(cfg, beta, fr.kl_per_feature * (n / B))
    integration, acts = fr.cache["integration"], fr.cache["int_acts"]
    Li = len(integration) - 1
    Wc, _ = integration[-1]
    dzs = weighted_dz(loss, fr.pred, y, sample_weight, B) * O.act_grad_from_output(cfg.output_activation_fn, fr.pred,
                                                                                  cfg.leaky_alpha)
    int_grads = [None] * (Li + 1)
    int_grads[Li] = np.concatenate([(acts[Li].T @ dzs).ravel(), dzs.sum(axis=0)])
    d = (S * dzs) @ Wc.T * Q._dact(cfg, acts[Li])
    for j in range(Li - 1, -1, -1):
        dg = R(d)
        W, _ = integration[j]
        int_grads[j] = np.concatenate([(acts[j].T @ dg).ravel() / S, d.sum(axis=0) / S])
        d = dg @ R(W).T
        if j > 0:
            d = d * Q._dact(cfg, acts[j])
    g_emb = R(d)
    fr.cache["d_emb16"] = g_emb
    enc = Q.encoder_backward(cfg, fr, eps, g_emb, beta_eff, B, S, fmt)
    _weigh(fr, loss, fr.pred, y, sample_weight, O.ib_loss(cfg, beta, fr.kl_per_feature))
    return np.concatenate([enc] + [g.ravel() for g in int_grads]), fr


# ---------------------------------------------------------------------------------------------------------------------
# tests/set_transformer_oracle.py and tests/set_transformer_varlen_oracle.py: one weight per set
# ---------------------------------------------------------------------------------------------------------------------
def set_transformer_train_grads(cfg, flat, x, y, eps, beta, loss, sample_weight, sizes=None):
    """STO.train_grads (sizes None) or VO.train_grads (padded sets of the given sizes) of the weighted loss."""
    if sizes is None:
        from tests import set_transformer_oracle as STO
        pred = STO.forward(cfg, flat, x, eps, beta).pred
        g, fr = STO.train_grads(cfg, flat, x, weighted_dz(loss, pred, y, sample_weight, x.shape[0]), eps, beta, "external")
    else:
        from tests import set_transformer_varlen_oracle as VO
        pred = VO.forward(cfg, flat, x, eps, sizes, beta).pred
        g, fr = VO.train_grads(cfg, flat, x, weighted_dz(loss, pred, y, sample_weight, x.shape[0]), eps, sizes, beta, "external")
    return g, _weigh(fr, loss, fr.pred, y, sample_weight, float(beta) * fr.kl)
