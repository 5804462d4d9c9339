"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the reference's InfoNCE training path (train.py:180-289) on top of
oracle/dib_oracle.py: the output encoder (train.py:186-193), the joint gradient of InfoNCE + beta * sum KL for the model
and the output encoder (train.py:198-220), and the fit loop with the full-batch plan of train.py:222-234.  A PyTorch
autograd twin of the output encoder sits beside it for cross-checks.  The product path never imports this module."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import dib_oracle as O
from oracle import torch_twin as TT


def output_encoder_layer_dims(cfg: O.DIBConfig, y_dimensionality, y_encoder_architecture):
    """train.py:186-193: Input(y_dim) -> [PositionalEncoding(2**arange(1, n))] -> Dense(h, act)... -> Dense(out)."""
    width = y_dimensionality * (1 + len(cfg.frequencies)) if cfg.use_positional_encoding else y_dimensionality
    return [width] + list(y_encoder_architecture) + [cfg.output_dimensionality]


def infonce_param_shapes(cfg: O.DIBConfig, y_dimensionality, y_encoder_architecture):
    """all_trainable_variables = model.trainable_variables + output_encoder.trainable_variables (train.py:198)."""
    d = output_encoder_layer_dims(cfg, y_dimensionality, y_encoder_architecture)
    shapes = list(cfg.param_shapes())
    for k in range(len(d) - 1):
        shapes += [(d[k], d[k + 1]), (d[k + 1],)]
    return shapes


def split_params(cfg: O.DIBConfig, flat, y_dimensionality, y_encoder_architecture):
    """-> (model flat params, output-encoder layers [(W, b), ...])."""
    flat = np.asarray(flat)
    px = flat[:cfg.param_count()]
    d = output_encoder_layer_dims(cfg, y_dimensionality, y_encoder_architecture)
    layers, off = [], cfg.param_count()
    for k in range(len(d) - 1):
        W = flat[off:off + d[k] * d[k + 1]].reshape(d[k], d[k + 1]); off += d[k] * d[k + 1]
        b = flat[off:off + d[k + 1]]; off += d[k + 1]
        layers.append((W, b))
    assert off == flat.size, (off, flat.size)
    return px, layers


def output_encoder_forward(cfg: O.DIBConfig, layers, y, keep=False):
    """train.py:186-193 (the same Sequential shape as an encoder, models.py:72-78, with a linear last Dense)."""
    y = np.asarray(y, dtype=np.float64)
    h = O.positional_encoding(y, cfg.frequencies) if cfg.use_positional_encoding else y
    acts = [h]
    for k, (W, b) in enumerate(layers):
        z = h @ W + b
        h = O.act_fwd(cfg.activation_fn, z, cfg.leaky_alpha) if k < len(layers) - 1 else z
        acts.append(h)
    return (h, acts) if keep else h


def infonce_loss_and_grads(e1, e2, similarity_type, temperature, chunk=64, want_grads=True):
    """O.infonce_loss_and_grads (train.py:203-213 and its reverse mode) evaluated in row blocks of `chunk`, so that the
    [n, n, d] pair tensors it forms are never whole: usable at a few thousand rows.  Returns (loss, d e1, d e2)."""
    a, b = np.asarray(e1, dtype=np.float64), np.asarray(e2, dtype=np.float64)
    n, T = a.shape[0], float(temperature)
    S = np.concatenate([O.get_scaled_similarity(a[i:i + chunk], b, similarity_type, T) for i in range(0, n, chunk)])
    row, col = O._logsumexp(S, 1), O._logsumexp(S, 0)
    loss = float((row - np.diag(S)).mean() + (col - np.diag(S)).mean())
    if not want_grads:
        return loss, None, None
    da, db = np.zeros_like(a), np.zeros_like(b)
    na, nb = np.linalg.norm(a, axis=-1), np.linalg.norm(b, axis=-1)
    for i0 in range(0, n, chunk):
        i1 = min(i0 + chunk, n)
        Sc = S[i0:i1]
        dS = (np.exp(Sc - row[i0:i1, None]) + np.exp(Sc - col[None, :])) / n
        dS[np.arange(i1 - i0), np.arange(i0, i1)] -= 2.0 / n
        diff = a[i0:i1, None, :] - b[None, :, :]
        if similarity_type == "l2sq":
            ga = -2.0 * diff / T
        elif similarity_type == "l2":
            ga = -diff / (-Sc * T)[:, :, None] / T
        elif similarity_type == "l1":
            ga = -np.sign(diff) / T
        elif similarity_type == "linf":
            k = np.abs(diff).argmax(-1)
            ga = np.zeros_like(diff)
            ii, jj = np.meshgrid(np.arange(i1 - i0), np.arange(n), indexing="ij")
            ga[ii, jj, k] = -np.sign(diff[ii, jj, k]) / T
        if similarity_type == "cosine":
            ah, bh = a[i0:i1] / na[i0:i1, None], b / nb[:, None]
            c = ah @ bh.T
            ga = (bh[None, :, :] - c[:, :, None] * ah[:, None, :]) / na[i0:i1, None, None] / T
            gb = (ah[:, None, :] - c[:, :, None] * bh[None, :, :]) / nb[None, :, None] / T
        else:
            gb = -ga
        da[i0:i1] = np.einsum("ij,ijk->ik", dS, ga)
        db += np.einsum("ij,ijk->jk", dS, gb)
    return loss, da, db


def infonce_train_grads(cfg: O.DIBConfig, params, x, y, eps, beta, *, y_dimensionality, y_encoder_architecture,
                        similarity="l2", temperature=1.0):
    """train.py:201-220 in float64: e1 = model(x), e2 = output_encoder(y), loss = InfoNCE(e1, e2) + beta * sum KL.
    Returns (flat gradient over all_trainable_variables, InfoNCE loss, KL per feature [F])."""
    px, layers = split_params(cfg, params, y_dimensionality, y_encoder_architecture)
    fr = O.forward(cfg, px, x, eps, beta, keep=False)
    e2, acts = output_encoder_forward(cfg, layers, y, keep=True)
    loss, d1, d2 = infonce_loss_and_grads(fr.pred, e2, similarity, temperature)
    gx, fr = O.train_grads(cfg, px, x, d1, eps, beta, "external")
    dz, gy = d2, [None] * len(layers)
    for k in reversed(range(len(layers))):
        W, _ = layers[k]
        gy[k] = (acts[k].T @ dz, dz.sum(axis=0))
        if k > 0:
            dz = (dz @ W.T) * O.act_grad_from_output(cfg.activation_fn, acts[k], cfg.leaky_alpha)
    flat = [gx] + [a.ravel() for g in gy for a in g]
    return np.concatenate(flat), float(loss), fr.kl_per_feature


def fit_infonce(cfg: O.DIBConfig, params, x, y, *, epochs, batch_size, lr, eps_fn, perm_fn, beta_fn=None,
                validation_data=None, val_perm_fn=None, y_dimensionality, y_encoder_architecture, similarity="l2",
                temperature=1.0):
    """Model.fit of an InfoNCE-compiled model: per epoch beta = beta_fn(epoch) (on_epoch_begin), floor(N/B) full batches of
    perm_fn(epoch, N), Adam over the joint buffer; validation floor(Nv/B) + 1 full batches of the repeated val_perm_fn(epoch,
    Nv).  eps_fn(step, rows) as O.fit: training keyed by (optimizer step, row in batch), validation by (2**31 + epoch,
    position in the repeated validation stream).  history: loss (InfoNCE + beta sum KL), KL{i}, beta and val_ twins."""
    p = np.array(params, dtype=np.float64, copy=True)
    st = O.AdamState(np.zeros_like(p), np.zeros_like(p))
    F = cfg.number_features
    hist = {k: [] for k in ["loss", "beta"] + [f"KL{i}" for i in range(F)]}
    if validation_data is not None:
        for k in list(hist):
            hist["val_" + k] = []
    kw = dict(y_dimensionality=y_dimensionality, y_encoder_architecture=y_encoder_architecture, similarity=similarity,
              temperature=temperature)
    N, B, step, beta = x.shape[0], batch_size, 0, 1.0
    assert N >= B
    for epoch in range(epochs):
        if beta_fn is not None:
            beta = float(beta_fn(epoch))
        perm = perm_fn(epoch, N)
        losses, kls = [], []
        for k in range(N // B):
            idx = perm[k * B:(k + 1) * B]
            g, loss, kl = infonce_train_grads(cfg, p, x[idx], y[idx], eps_fn(step, np.arange(B)), beta, **kw)
            O.adam_step(p, g, st, lr)
            losses.append(loss + beta * kl.sum()); kls.append(kl)
            step += 1
        hist["loss"].append(float(np.mean(losses))); hist["beta"].append(beta)
        for i in range(F):
            hist[f"KL{i}"].append(float(np.mean([k_[i] for k_ in kls])))
        if validation_data is not None:
            xv, yv = validation_data
            Nv = xv.shape[0]
            vperm = val_perm_fn(epoch, Nv)
            losses, kls = [], []
            for k in range(Nv // B + 1):
                pos = np.arange(k * B, (k + 1) * B)
                idx = vperm[pos % Nv]
                px, layers = split_params(cfg, p, y_dimensionality, y_encoder_architecture)
                fr = O.forward(cfg, px, xv[idx], eps_fn(2 ** 31 + epoch, pos), beta)
                e2 = output_encoder_forward(cfg, layers, yv[idx])
                loss = infonce_loss_and_grads(fr.pred, e2, similarity, temperature, want_grads=False)[0]
                losses.append(loss + beta * fr.kl_per_feature.sum()); kls.append(fr.kl_per_feature)
            hist["val_loss"].append(float(np.mean(losses))); hist["val_beta"].append(beta)
            for i in range(F):
                hist[f"val_KL{i}"].append(float(np.mean([k_[i] for k_ in kls])))
    return p, hist


# ---------------------------------------------------------------------------------------------------------------------
# autograd twin
# ---------------------------------------------------------------------------------------------------------------------
class TwinOutputEncoder(torch.nn.Module):
    """train.py:186-193 as a torch Sequential (PositionalEncoding -> Linear/act ... -> Linear)."""

    def __init__(self, cfg: O.DIBConfig, y_dimensionality, y_encoder_architecture):
        super().__init__()
        dims = output_encoder_layer_dims(cfg, y_dimensionality, y_encoder_architecture)
        layers = [TT.PositionalEncoding(cfg.frequencies)] if cfg.use_positional_encoding else []
        for k in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[k], dims[k + 1]))
            if k < len(dims) - 2:
                layers.append(TT._ACT[cfg.activation_fn]())
        self.net = torch.nn.Sequential(*layers)

    def linears(self):
        return [m for m in self.net if isinstance(m, torch.nn.Linear)]

    def forward(self, y):
        return self.net(y)


def torch_similarity(a, b, similarity_type, temperature):
    """utils.py:75-175 in torch (the reference's forms, autograd-differentiable)."""
    if similarity_type in ("l2sq", "l2"):
        d2 = torch.clamp((a * a).sum(-1)[:, None] + (b * b).sum(-1)[None, :] - 2.0 * a @ b.T, min=0.0)
        sim = -d2 if similarity_type == "l2sq" else -torch.sqrt(d2 + 1e-9)
    elif similarity_type == "l1":
        sim = -(a[:, None, :] - b[None, :, :]).abs().sum(-1)
    elif similarity_type == "linf":
        sim = -(a[:, None, :] - b[None, :, :]).abs().amax(-1)
    else:
        sim = torch.nn.functional.normalize(a, dim=-1) @ torch.nn.functional.normalize(b, dim=-1).T
    return sim / temperature


def torch_infonce(e1, e2, similarity_type, temperature):
    S = torch_similarity(e1, e2, similarity_type, temperature)
    lab = torch.arange(S.shape[0])
    return torch.nn.functional.cross_entropy(S, lab) + torch.nn.functional.cross_entropy(S.T, lab)


def twin_infonce_grads(cfg: O.DIBConfig, params, x, y, eps, beta, *, y_dimensionality, y_encoder_architecture,
                       similarity="l2", temperature=1.0):
    """The same gradient as infonce_train_grads by autograd through TwinDIB + TwinOutputEncoder (float64)."""
    px, _ = split_params(cfg, params, y_dimensionality, y_encoder_architecture)
    model = TT.TwinDIB(cfg).double()
    model.load_flat(px)
    enc = TwinOutputEncoder(cfg, y_dimensionality, y_encoder_architecture).double()
    off = cfg.param_count()
    flat = np.asarray(params, dtype=np.float64)
    with torch.no_grad():
        for lin in enc.linears():
            fi, fo = lin.in_features, lin.out_features
            lin.weight.copy_(torch.from_numpy(flat[off:off + fi * fo].reshape(fi, fo).T.copy())); off += fi * fo
            lin.bias.copy_(torch.from_numpy(flat[off:off + fo].copy())); off += fo
    pred, kls = model(torch.from_numpy(np.asarray(x, np.float64)), torch.from_numpy(np.asarray(eps, np.float64)))
    e2 = enc(torch.from_numpy(np.asarray(y, np.float64)))
    loss = torch_infonce(pred, e2, similarity, temperature)
    (loss + beta * kls.sum()).backward()
    g = [model.flat_grads()] + [t for lin in enc.linears() for t in (lin.weight.grad.T.reshape(-1), lin.bias.grad.reshape(-1))]
    return torch.cat(g).numpy(), float(loss.detach())


def glorot(shapes, rng):
    out = []
    for s in shapes:
        if len(s) == 2:
            lim = math.sqrt(6.0 / (s[0] + s[1]))
            out.append(rng.uniform(-lim, lim, size=s).ravel())
        else:
            out.append(rng.standard_normal(s) * 0.05)
    return np.concatenate(out)
