"""TEST INFRASTRUCTURE ONLY -- a float64 reference of the fused per-feature encoder kernels of the 'fp16' / 'bf16' precision
(csrc/dib_enc_fused.cu: dib_enc_pack_weights_kernel, dib_enc_fused_fwd_kernel and dib_enc_fused_bwd_kernel), per 128-row
tile and per (feature, slot), rounding exactly where the kernels round.  Not collected by pytest (no test_ prefix).

Exactness (the exact regime).  relu, leaky ReLU with alpha = 1/4 and linear; dyadic x, weights, eps and d emb; a zero
logvar: W2's logvar columns 0 and b2's logvar half -logvar_offset, so that the packed carrier fl32(b2 + logvar_offset) is 0,
lv = 0 and both __expf(0) (forward) and expf(0) (backward) are 1.  Then every accumulator holds an exact sum (asserted with
``fp_exact.fits`` on the terms' magnitudes, for the weight gradients over every tile one slot accumulates) and every
fp32 epilogue operation is restated in numpy float32, one operation per kernel operation:
  pack (:913-945)              W0p [16][128] = W0 rows k < w_in, b0 in row w_in, 0 below; W1; W2; Bb1 [16][128] = b1 in row
                               w_in; Bb2 [16][64] = fl32(b2 + logvar_offset (logvar half)) in row w_in -- each r() saturating
  [pe | 1] (write_a0_row :242-264) column k < w_in = blk d + j: x_j (blk 0) or r(dib_sin_pe(2^blk x_j)); column w_in = 1
                               on rows inside the batch, 0 past it; the rest 0
  layers (:357-390)            h1 = r(act(a0 W0p)); h2 = r(act(a0 Bb1 + h1 W1)); (mu | lv) = a0 Bb2 + h2 W2; leaky ReLU
                               forms fl32(alpha z) before r() (dib_act16); relu is cvt.rn.relu (frag_to_a :163-172)
  forward epilogue (:486-507)  sv = __expf(0.5 lv); u = fma(sv, eps, mu); KL term 0.5 (mu mu + sv sv - lv - 1) added to the
                               thread's sum; emb = TF32(u) (cvt.rna), user_emb = u, emb16 = r(u); rows past n skipped
  KL partial (:509-517)        kl_part[f, slot] = the sum over the slot's tiles and rows < n (exact: the order is free)
  backward dO (:743-785)       g = fl32(d_emb S) or the d_emb16 value; bs = fl32(fl32(beta inv_batch) S);
                               dm = fma(bs, mu, g); dl = fma(fl32(g eps), 0.5 sgm, bs 0.5 (sgm sgm - 1)), sgm = expf(0.5 lv);
                               dO = r([dm | dl]) and 0 past n
  dgrad (:201-223, :791-853)   dz2 = r(G2) (h2 > 0) for relu (the gate is taken from the ROUNDED h2), r(fl32(G2 act'(h2)))
                               otherwise, G2 = dO W2^T; dz1 likewise from G1 = dz2 W1^T and h1
  weight gradients (:791-906)  per (feature, slot) over the slot's tiles: dW2 = h2^T dO, db2 = dO^T 1, dW1 = h1^T dz2,
                               db1 = dz2^T 1, [dW0; db0] = dz1^T [pe | 1] (column w_in is db0), each fl32(acc (1 / S)); the
                               weight-gradient accumulators restart (scale-d = 0) at each feature's first tile (wacc)
  schedule (sched_of :409-415) grid G >= F: CTA c serves feature c % F, slot c / F, tiles slot, slot + nslots, ... with
                               nslots = ceil((G - f) / F); G < F: CTA c walks features c, c + G, ... with all their tiles
                               in slot 0.

r() is ``fp_exact.round_to``: half to even, saturating (cvt.rn.satfinite).

Bounded regime (``bounded_forward`` / ``bounded_backward``): lv != 0, tanh / sigmoid / elu, leaky ReLU with alpha = 0.2, and any
sum that does not fit 24 bits.  Every value is the float64 function of the reference's own float64 intermediates, with a
first-order bound e on its distance from the kernel's value, multiplied by ``fp_exact.C_BOUND`` at the outputs:
  * SFU activations: ``int16_reference.act16`` (tanh.approx 2^-10.987 relative, ex2.approx 2^-22 relative plus the rounding
    of its argument) and one 16-bit ulp; |act'| <= 1 carries the pre-activation's error through; leaky ReLU / relu / linear
    restate fl32(alpha z) and r() and add one 16-bit ulp wherever the pre-activation is inexact.
  * h1, h2, dz2 and dz1 never leave the chip: a contraction of inexact operands is bounded by |W| e + tc_gamma(K) |a| |W|
    (the tensor core's fp32 sums may truncate on alignment: 2u per add); act'(h) from an inexact h by its derivative (tanh
    2 |h| e, sigmoid |1 - 2 h| e, elu e) and, for relu / leaky ReLU, 1 - alpha where |h| <= e (the gate may flip).
  * forward epilogue: sv = __expf(0.5 lv): sv (e_lv / 2 + 2^-22 + |lv| u + u); u = fma(sv, eps, mu): |eps| e_sv + e_mu + u |u|;
    KL term: |mu| e_mu + sv e_sv + e_lv / 2 + 2u (mu^2 + sv^2 + |lv| + 1); kl_part: the terms' bounds plus gamma_m sum |terms|.
    emb adds half a TF32 ulp (2^-11 |u|), emb16 one 16-bit ulp.
  * backward epilogue: sgm = expf(0.5 lv) (libm, 2 ulp): sgm (e_lv / 2 + 5u); dm = fma(bs, mu, g): bs e_mu + u |dm|;
    dl = fma(fl(g eps), fl(0.5 sgm), bs 0.5 fl(sgm sgm - 1)) -- contracted or not, within |g eps| e_sgm / 2 + 3u |g eps sgm| / 2
    + bs (sgm e_sgm + u (sgm^2 + 1)) + u |dl|; dO adds one 16-bit ulp.
  * weight gradients: e_a^T |b| + |a|^T e_b + tc_gamma(rows) |a|^T |b| per (feature, slot).
  * dib_sin_pe: sin.approx.f32 of the reduced argument (PTX ISA: 2^-20.5 absolute on [-pi, pi]) plus the reduction: k C1
    is subtracted exactly, the second fma rounds once (2^-23 at |r| <= pi) and C2's own rounding adds |k| |C2| 2^-24
    (below 2^-28 for |a| < 2^17).  SIN_TOL = 2^-20.5 + 2^-22 covers both.
  * the Philox noise against oracle/philox.normal_noise: ``elementwise_reference.Z_TOL`` (1 + |z|), set there from
    measurement.
Two readout networks turn on-chip values into exact outputs: ``pe_readout_params`` routes every [pe | 1] column to a mu column
(relu: +-relu pairs; linear: the identity), so with eps = 0 emb16 is the kernel's 16-bit first-layer operand; ``noise
readout`` (W2 = 0, b2 = 0) makes u the noise itself.

``fault`` arguments seed one kernel fault each into the restatement (tests/test_enc_fused_reference_host.py shows each one
breaks a comparison); None is the kernel."""
from __future__ import annotations

import numpy as np

from tests import elementwise_reference as ER
from tests import int16_reference as I
from tests.fp_exact import (C_BOUND, EXACT_BITS, U, dyadic, exact_matmul, f32, fits, gamma, quantum, r16, round_tf32,
                             sparse_dyadic, ulp16)

TM, HID, EO, K0, E = 128, 128, 64, 16, 32
PACK_ELEMS = K0 * HID + HID * HID + HID * EO + K0 * HID + K0 * EO
ACTS = ER.ACTS
Z_TOL = ER.Z_TOL
SIN_TOL = 2.0 ** -20.5 + 2.0 ** -22
BLOCKS = ("w0", "b0", "w1", "b1", "w2", "b2")


def _has(fault, name):
    """fault is None, one fault name or a tuple of them"""
    return fault == name or (isinstance(fault, tuple) and name in fault)


# ---- parameter layout -----------------------------------------------------------------------------------------------------
def layout(fdims, nfreq, gap=0):
    """Offsets of each feature's [W0 (w_in x 128), b0, W1, b1, W2, b2] in the model's order, ``gap`` floats apart.
    Returns (dict block -> int64 [F], total count)."""
    off = {b: [] for b in BLOCKS}
    pos = 0
    for d in fdims:
        for b, size in zip(BLOCKS, (d * nfreq * HID, HID, HID * HID, HID, HID * EO, EO)):
            off[b].append(pos)
            pos += size + gap
    return {b: np.asarray(v, np.int64) for b, v in off.items()}, pos


def flatten_params(enc, lay, count):
    p = np.zeros(count)
    for f, e in enumerate(enc):
        for b, k in zip(BLOCKS, ("W0", "b0", "W1", "b1", "W2", "b2")):
            v = np.asarray(e[k], np.float64).ravel()
            p[int(lay[b][f]):int(lay[b][f]) + v.size] = v
    return p


# ---- the pack ---------------------------------------------------------------------------------------------------------------
def pack(enc, fdims, nfreq, logvar_offset, fmt, fault=None):
    """The 16-bit image [F, PACK_ELEMS] (float64 values) of dib_enc_pack_weights_kernel."""
    out = np.zeros((len(fdims), PACK_ELEMS))
    for f, (e, d) in enumerate(zip(enc, fdims)):
        w_in = d * nfreq
        w0p = np.zeros((K0, HID))
        w0p[:w_in] = e["W0"]
        w0p[w_in] = e["b0"]
        bb1 = np.zeros((K0, HID))
        bb1[w_in] = e["b1"]
        bb2 = np.zeros((K0, EO))
        off = np.concatenate([np.zeros(E), np.full(E, np.float32(logvar_offset), np.float64)])
        bb2[w_in] = f32(f32(e["b2"]) + f32(off)).astype(np.float64)            # :941 one fp32 add, then r()
        img = np.concatenate([w0p.ravel(), np.asarray(e["W1"]).ravel(), np.asarray(e["W2"]).ravel(), bb1.ravel(), bb2.ravel()])
        out[f] = r16(img, fmt)
        if _has(fault, "offset_after_round"):
            out[f, -K0 * EO + w_in * EO:-K0 * EO + (w_in + 1) * EO] = r16(e["b2"], fmt) + off
    return out


def split_pack(img):
    """One feature's image -> (W0p [16, 128], W1, W2, Bb1 [16, 128], Bb2 [16, 64])."""
    a = K0 * HID
    b = a + HID * HID
    c = b + HID * EO
    d = c + K0 * HID
    return (img[:a].reshape(K0, HID), img[a:b].reshape(HID, HID), img[b:c].reshape(HID, EO), img[c:d].reshape(K0, HID),
            img[d:].reshape(K0, EO))


# ---- the schedule -----------------------------------------------------------------------------------------------------------
def schedule(F, grid, tiles, fault=None):
    """sched_of: [(cta, feature, slot, [tiles])] in each CTA's order.  fault 'slot_count': one slot too many per feature
    (tiles credited to the wrong slot); 'wrong_slot': the second tile of a multi-tile slot credited to the next slot."""
    out = []
    for c in range(grid):
        if grid >= F:
            f0, slot = c % F, c // F
            nslots = (grid - f0 + F - 1) // F + (1 if _has(fault, "slot_count") else 0)
            ts = list(range(slot, tiles, nslots))
            out.append((c, f0, slot, ts))
        else:
            for f in range(c, F, grid):
                out.append((c, f, 0, list(range(tiles))))
    if _has(fault, "wrong_slot"):                                        # the first multi-tile slot loses its second tile
        k = next(i for i, (_, _, _, ts) in enumerate(out) if len(ts) > 1)
        c, f, s, ts = out[k]
        out[k:k + 1] = [(c, f, s, [ts[0]] + ts[2:]), (c, f, s + 1, [ts[1]])]
    return out


def slots_per_feature(F, grid):
    """The slot rows each feature writes (the kl_part entries and the partial rows)."""
    return [(grid - f + F - 1) // F if grid >= F else 1 for f in range(F)]


# ---- the first-layer operand -----------------------------------------------------------------------------------------------
def pe_columns(d, nfreq):
    """(source column j, frequency 2^blk or 0 for the plain x) of each first-layer column k < d nfreq."""
    return [(k % d, 0 if k // d == 0 else 2 ** (k // d)) for k in range(d * nfreq)]


def sin_values(xf, d, nfreq, fault=None):
    """sin(fl32(2^blk) fl32(x_j)) in float64 for every PE column (the plain columns hold x), [rows, w_in]."""
    xf = np.asarray(xf, np.float32).astype(np.float64)
    cols = []
    for j, fr in pe_columns(d, nfreq):
        if fr == 0:
            cols.append(xf[:, j])
        else:
            cols.append(np.sin((2 * fr if _has(fault, "freq") else fr) * xf[:, j]))
    return np.stack(cols, 1) if cols else np.zeros((xf.shape[0], 0))


def near_midpoint(s, fmt, margin):
    """True where s lies within ``margin`` of a rounding midpoint of fmt (or of a boundary where r() changes)."""
    return (r16(s - margin, fmt) != r16(s + margin, fmt))


def a0_operand(xf, n_valid, d, nfreq, fmt, fault=None):
    """[pe | 1 | 0] [rows, 16] (16-bit values) of write_a0_row for rows 0 .. rows - 1 (rows >= n_valid: the batch end, where
    x reads as 0 and the ones column is 0).  Exact where the sine values lie farther than SIN_TOL from a midpoint (the caller
    asserts that with ``pe_exact``)."""
    xf = np.asarray(xf, np.float32).astype(np.float64)
    rows = xf.shape[0]
    valid = np.arange(rows) < n_valid
    xz = np.where(valid[:, None], xf, 0.0)
    w_in = d * nfreq
    a = np.zeros((rows, K0))
    a[:, :w_in] = r16(sin_values(xz, d, nfreq, fault), fmt)
    a[:, w_in] = 1.0 if _has(fault, "ones_past_n") else valid.astype(np.float64)
    return a


def pe_exact(xf, d, nfreq, fmt):
    """True where every sine column of these rows lies farther than SIN_TOL from a rounding midpoint of fmt."""
    s = sin_values(xf, d, nfreq)
    k = np.array([fr != 0 for _, fr in pe_columns(d, nfreq)], bool)
    return ~near_midpoint(s[:, k], fmt, SIN_TOL).any(1) if k.any() else np.ones(s.shape[0], bool)


# ---- activations ------------------------------------------------------------------------------------------------------------
def act16(act, z, alpha, fmt):
    """r(dib_act16(act, z)) for the exact activations from the exact fp32 accumulator z (float64 values)."""
    z32 = f32(z)
    if act == "relu":
        return r16(np.maximum(z, 0.0), fmt)
    if act == "leaky_relu":
        return r16(np.where(z32 > 0, z32, np.float32(alpha) * z32).astype(np.float64), fmt)
    assert act == "linear", f"{act}: the exact reference takes relu, leaky_relu or linear"
    return r16(z, fmt)


def exact_act_grad32(act, h, alpha):
    return np.where(h > 0, np.float32(1), np.float32(alpha)).astype(np.float32) if act == "leaky_relu" else (
        (h > 0).astype(np.float32) if act == "relu" else np.ones(np.shape(h), np.float32))


def dgrad16(act, G, h, alpha, fmt):
    """dz = r(G) gated by h > 0 (relu: relu_gate2 of the rounded h) or r(fl32(G act'(h)))."""
    if act == "relu":
        return r16(G, fmt) * (h > 0)
    return r16((f32(G) * exact_act_grad32(act, h, alpha)).astype(np.float64), fmt)


# ---- one feature, all rows ---------------------------------------------------------------------------------------------------
def feature_chain(img, xf, n, d, nfreq, act, alpha, fmt, fault=None):
    """The on-chip forward chain of one feature over ceil(n / 128) whole tiles: a0, h1, h2, mu, lv [tiles 128, ...]."""
    rows = -(-n // TM) * TM
    xp = np.zeros((rows, d), np.float32)
    xp[:n] = np.asarray(xf, np.float32)[:n]
    W0p, W1, W2, Bb1, Bb2 = split_pack(img)
    a0 = a0_operand(xp, n, d, nfreq, fmt, fault)
    z1 = exact_matmul(a0, W0p, "layer 0")
    h1 = act16(act, z1, alpha, fmt)
    if _has(fault, "no_bias_carrier"):                                         # the K = 16 bias-carrier step dropped
        z2 = exact_matmul(h1, W1, "layer 1")
        h2 = act16(act, z2, alpha, fmt)
    elif _has(fault, "bias_after_act"):                                        # b1 added after the activation
        z2 = exact_matmul(h1, W1, "layer 1")
        h2 = r16(act16(act, z2, alpha, fmt) + a0 @ Bb1, fmt)
    else:
        z2 = exact_matmul(np.concatenate([a0, h1], 1), np.concatenate([Bb1, W1], 0), "layer 1 + bias carrier")
        h2 = act16(act, z2, alpha, fmt)
    o = exact_matmul(np.concatenate([a0, h2], 1), np.concatenate([Bb2, W2], 0), "layer 2 + bias carrier")
    return dict(a0=a0, h1=h1, h2=h2, pre1=z1, pre2=z2, mu=o[:, :E], lv=o[:, E:])


def _noise_rows(eps, f, rows, n):
    z = np.zeros((rows, E))
    z[:n] = np.asarray(eps, np.float64)[:n, f, :]
    return z


def forward(img_all, x, x_off, fdims, nfreq, act, alpha, fmt, n, eps, grid, fault=None):
    """The forward kernel's outputs in the exact regime: emb (TF32), user_emb, emb16 [n, 32 F] and kl_part [F, slots]
    (float64), plus the per-feature chains (for the backward)."""
    F = len(fdims)
    tiles = -(-n // TM)
    user = np.zeros((n, E * F))
    chains = []
    sched = schedule(F, grid, tiles, fault)
    kl = np.zeros((F, max(s for _, _, s, _ in sched) + 1))
    for f, d in enumerate(fdims):
        xf = np.asarray(x, np.float32)[:n, x_off[f]:x_off[f] + d]
        ch = feature_chain(img_all[f], xf, n, d, nfreq, act, alpha, fmt, fault)
        assert np.all(ch["lv"] == 0), "the exact reference needs lv = 0 (W2's logvar columns 0, b2's logvar half -offset)"
        z = _noise_rows(eps, f, tiles * TM, n)
        mu = ch["mu"]
        fits(np.abs(z) + np.abs(mu), min(quantum(z), quantum(mu)), "u = fma(sv, eps, mu)")
        u = z + mu                                                          # sv = __expf(0) = 1
        user[:, f * E:(f + 1) * E] = u[:n]
        term = 0.5 * mu * mu                                                # 0.5 (mu mu + 1 - 0 - 1)
        fits(mu * mu + 1.0, quantum(mu) ** 2, "KL term mu mu + sv sv")
        ch["kl_rows"] = term.sum(1) if _has(fault, "kl_past_n") else np.where(np.arange(tiles * TM) < n, term.sum(1), 0.0)
        chains.append(ch)
    for c, f, s, ts in sched:
        rows = np.concatenate([np.arange(t * TM, (t + 1) * TM) for t in ts]) if ts else np.zeros(0, int)
        v = chains[f]["kl_rows"][rows]
        fits(np.abs(v).sum(), quantum(v) if v.size else 1.0, "KL partial")
        kl[f, s] = v.sum()
    return dict(user_emb=user, emb=round_tf32(f32(user)).astype(np.float64), emb16=r16(user, fmt), kl_part=kl, chains=chains)


def backward(img_all, chains, fdims, nfreq, act, alpha, fmt, n, eps, g, beta, inv_batch, S, grid, lay, fault=None):
    """The backward kernel's weight-gradient partials in the exact regime: {(feature, slot): {block: array}} from
    g [n, 32 F] = the S-scaled gradient as the kernel reads it (fl32(d_emb S) or the d_emb16 value)."""
    F = len(fdims)
    tiles = -(-n // TM)
    rows_all = tiles * TM
    bs = float(f32(f32(np.float32(beta) * np.float32(inv_batch)) * np.float32(S)))
    if fault == "bs_without_S":
        bs = float(f32(np.float32(beta) * np.float32(inv_batch)))
    valid = np.arange(rows_all) < n
    per_feature = []
    for f, d in enumerate(fdims):
        ch = chains[f]
        W0p, W1, W2, _, _ = split_pack(img_all[f])
        gf = np.zeros((rows_all, E))
        gf[:n] = g[:n, f * E:(f + 1) * E]
        z = _noise_rows(eps, f, rows_all, n)
        mu = ch["mu"]
        bsv = np.where(valid, bs, 0.0)[:, None]
        dm = f32(bsv * mu + gf).astype(np.float64)                         # fma: the float64 value is exact, one rounding
        gz = f32(gf * z).astype(np.float64)
        dl = gz * (1.0 if _has(fault, "dl_without_half") else 0.5)              # + bs 0.5 (1 - 1) = +0
        dO = r16(np.concatenate([dm, dl], 1), fmt)
        dO[~valid] = 0.0
        # the relu gate reads the rounded h (fault: the fp32 pre-activation, which differs where r() flushes it to 0)
        gate = (lambda k: ch["pre" + k]) if _has(fault, "gate_unrounded") else (lambda k: ch["h" + k])
        G2 = exact_matmul(dO, W2.T, "G2")
        dz2 = dgrad16(act, G2, gate("2"), alpha, fmt)
        G1 = exact_matmul(dz2, W1.T, "G1")
        dz1 = dgrad16(act, G1, gate("1"), alpha, fmt)
        per_feature.append(dict(a0=ch["a0"], h1=ch["h1"], h2=ch["h2"], dO=dO, dz2=dz2, dz1=dz1))
    out = {}
    prev = {}
    inv_s = float(np.float32(1.0) / np.float32(S))
    for c, f, s, ts in schedule(F, grid, tiles, fault):
        pf = per_feature[f]
        rows = np.concatenate([np.arange(t * TM, (t + 1) * TM) for t in ts])
        a0, h1, h2, dO, dz2, dz1 = (pf[k][rows] for k in ("a0", "h1", "h2", "dO", "dz2", "dz1"))
        acc = dict(w2=exact_matmul(h2.T, dO, "dW2"), b2=exact_matmul(a0.T, dO, "db2")[fdims[f] * nfreq],
                   w1=exact_matmul(h1.T, dz2, "dW1"), b1=exact_matmul(a0.T, dz2, "db1")[fdims[f] * nfreq],
                   w0p=exact_matmul(dz1.T, a0, "dW0p^T"))
        if _has(fault, "no_restart") and c in prev and prev[c][0] != f:
            for k in ("w2", "b2", "w1", "b1"):
                acc[k] = acc[k] + prev[c][1][k]
        prev[c] = (f, acc)
        w_in = fdims[f] * nfreq
        blocks = dict(w0=acc["w0p"][:, :w_in].T.ravel(), b0=acc["w0p"][:, w_in], w1=acc["w1"].ravel(), b1=acc["b1"],
                      w2=acc["w2"].ravel(), b2=acc["b2"])
        if _has(fault, "db0_unrouted"):                                   # col == w_in of dW0 not routed to db0
            blocks["b0"] = np.zeros(HID)
        if _has(fault, "db2_both"):                                       # warpgroup 1 stores its copy 64 floats further
            blocks["b2"] = np.concatenate([blocks["b2"], blocks["b2"]])
        out[(f, s)] = {k: (f32(v) * np.float32(inv_s)).astype(np.float64) for k, v in blocks.items()}
    return out


def partial_table(parts, lay, split_stride, nslots, sentinel):
    """The partial rows [nslots, split_stride] the backward leaves: every written block, the sentinel elsewhere."""
    t = np.full((nslots, split_stride), sentinel, np.float64)
    for (f, s), blocks in parts.items():
        for b, v in blocks.items():
            o = int(lay[b][f])
            t[s, o:o + v.size] = v
    return t


# ---- generators -------------------------------------------------------------------------------------------------------------
def exact_params(rng, fdims, nfreq, logvar_offset, density=1 / 16):
    """Encoder parameters with lv = 0 on coarse grids, so that every sum fits 24 bits over thousands of rows: weights in
    {-1, 0, 1} (W1 and W2 sparse), biases on the grid 1/2; W2's logvar columns 0 and b2's logvar half -fl32(logvar_offset)."""
    enc = []
    for d in fdims:
        w_in = d * nfreq
        W2 = sparse_dyadic(rng, (HID, EO), 1, 1, density)
        W2[:, E:] = 0.0
        b2 = dyadic(rng, EO, 2, 2)
        b2[E:] = -float(np.float32(logvar_offset))
        enc.append(dict(W0=dyadic(rng, (w_in, HID), 1, 1), b0=dyadic(rng, HID, 2, 2),
                        W1=sparse_dyadic(rng, (HID, HID), 1, 1, density), b1=dyadic(rng, HID, 2, 2), W2=W2, b2=b2))
    return enc


def pe_readout_params(fdims, nfreq, act):
    """0 / +-1 weights that route every [pe | 1] column k <= w_in to mu column k (eps = 0 makes emb16 the operand): relu
    through the pair relu(a) - relu(-a), linear through the identity.  b2 = 0, logvar 0 (with logvar_offset = 0)."""
    assert act in ("relu", "linear")
    enc = []
    for d in fdims:
        w_in = d * nfreq
        W0, b0, W1, W2 = np.zeros((w_in, HID)), np.zeros(HID), np.zeros((HID, HID)), np.zeros((HID, EO))
        for k in range(w_in + 1):
            col = W0[k] if k < w_in else b0
            if act == "relu":
                col[2 * k], col[2 * k + 1] = 1.0, -1.0
                W1[2 * k, 2 * k] = W1[2 * k + 1, 2 * k + 1] = 1.0
                W2[2 * k, k], W2[2 * k + 1, k] = 1.0, -1.0
            else:
                col[k] = 1.0
                W1[k, k] = 1.0
                W2[k, k] = 1.0
        enc.append(dict(W0=W0, b0=b0, W1=W1, b1=np.zeros(HID), W2=W2, b2=np.zeros(EO)))
    return enc


def noise_readout_params(rng, fdims, nfreq):
    """W2 = 0 and b2 = 0: mu = lv = 0, so u is the noise itself (the hidden layers are arbitrary)."""
    enc = exact_params(rng, fdims, nfreq, 0.0)
    for e in enc:
        e["W2"][:] = 0.0
        e["b2"][:] = 0.0
    return enc


def philox_noise(seed, step, sample_offset, n, F, fault=None):
    """oracle/philox.normal_noise of rows sample_offset + r, float64 [n, F, 32].  fault 'row_key': keyed by r alone;
    'swap_quad': dims 4 q + 1 and 4 q + 2 exchanged."""
    from oracle.philox import normal_noise
    ids = np.arange(n, dtype=np.uint64) + (np.uint64(0) if _has(fault, "row_key") else np.uint64(sample_offset))
    z = normal_noise(seed, step, ids, F, E, dtype=np.float64)
    if _has(fault, "swap_quad"):
        z = z.copy()
        z[..., 1::4], z[..., 2::4] = z[..., 2::4].copy(), z[..., 1::4].copy()
    return z


# ---- the bounded regime -------------------------------------------------------------------------------------------------
def _fit(a, b):
    """True when every sum of a @ b is exact in fp32 in any order (the 24-bit fit of int16_reference.fits)."""
    m = float(np.max(np.abs(a) @ np.abs(b), initial=0.0)) / (quantum(a) * quantum(b))
    return m < 2.0 ** EXACT_BITS


def mm_bounded(a, ea, b, eb=None):
    """a @ b and the bound of the kernel's fp32 (tensor-core) contraction of operands within ea / eb of a / b."""
    v = a @ b
    eb = np.zeros_like(b) if eb is None else eb
    if not ea.any() and not eb.any() and _fit(a, b):
        return v, np.zeros_like(v)
    return v, ea @ np.abs(b) + np.abs(a) @ eb + I.tc_gamma(a.shape[1]) * (np.abs(a) @ np.abs(b))


def act_bounded(act, z, ez, alpha, fmt):
    """The 16-bit activation of a pre-activation z known to within ez: (reference value, bound)."""
    if act in ("relu", "linear", "leaky_relu"):
        if not ez.any() and np.array_equal(f32(z).astype(np.float64), z):
            return act16(act, z, alpha, fmt), np.zeros_like(z)
        v = np.where(z > 0, z, (0.0 if act == "relu" else (1.0 if act == "linear" else alpha)) * z)
        e = ez + U * np.abs(z)
        return v, e + ulp16(np.abs(v) + e, fmt)
    v, e = I.act16(act, f32(z), alpha, fmt)
    z32 = f32(z).astype(np.float64)
    return np.asarray(v, np.float64), e + ez + np.abs(z32 - z)            # |act'| <= 1


def act_grad_bounded(act, h, eh, alpha):
    """dib_act_grad from the 16-bit h (reference h within eh): (value, bound)."""
    if act in ("relu", "leaky_relu"):
        lo = 0.0 if act == "relu" else float(np.float32(alpha))
        v = np.where(h > 0, 1.0, lo)
        return v, np.where((eh > 0) & (np.abs(h) <= eh), 1.0 - lo, 0.0)
    if act == "linear":
        return np.ones_like(h), np.zeros_like(h)
    if act == "tanh":
        return 1.0 - h * h, 2 * np.abs(h) * eh + eh * eh + 2 * U
    if act == "sigmoid":
        return h * (1.0 - h), np.abs(1.0 - 2 * h) * eh + eh * eh + 2 * U
    if act == "elu":
        return np.where(h > 0, 1.0, h + 1.0), eh + U
    raise ValueError(act)


def _r16_bound(v, e, fmt):
    return np.where(e > 0, e + ulp16(np.abs(v) + e, fmt), 0.0)


def bounded_forward(img_all, x, x_off, fdims, nfreq, act, alpha, fmt, n, eps, grid):
    """The forward kernel's outputs with bounds: emb, user_emb, emb16 [n, 32 F], kl_part [F, slots] and their *_bound,
    plus the per-feature chains for ``bounded_backward``.  eps is explicit (exact)."""
    F = len(fdims)
    tiles = -(-n // TM)
    rows_all = tiles * TM
    user, user_b = np.zeros((n, E * F)), np.zeros((n, E * F))
    chains = []
    for f, d in enumerate(fdims):
        xp = np.zeros((rows_all, d), np.float32)
        xp[:n] = np.asarray(x, np.float32)[:n, x_off[f]:x_off[f] + d]
        W0p, W1, W2, Bb1, Bb2 = split_pack(img_all[f])
        a0 = a0_operand(xp, n, d, nfreq, fmt)
        z0 = np.zeros_like(a0)
        z1, e1 = mm_bounded(a0, z0, W0p)
        h1, eh1 = act_bounded(act, z1, e1, alpha, fmt)
        z2, e2 = mm_bounded(np.concatenate([a0, h1], 1), np.concatenate([z0, eh1], 1), np.concatenate([Bb1, W1], 0))
        h2, eh2 = act_bounded(act, z2, e2, alpha, fmt)
        o, eo = mm_bounded(np.concatenate([a0, h2], 1), np.concatenate([z0, eh2], 1), np.concatenate([Bb2, W2], 0))
        mu, lv, emu, elv = o[:, :E], o[:, E:], eo[:, :E], eo[:, E:]
        sv = np.exp(0.5 * lv)
        e_sv = sv * (0.5 * elv + I.EX2_APPROX_REL + np.abs(lv) * U + U)
        z = _noise_rows(eps, f, rows_all, n)
        u = sv * z + mu
        e_u = np.abs(z) * e_sv + emu + U * np.abs(u)
        user[:, f * E:(f + 1) * E], user_b[:, f * E:(f + 1) * E] = u[:n], e_u[:n]
        term = 0.5 * (mu * mu + np.expm1(lv) - lv)
        e_t = np.abs(mu) * emu + sv * e_sv + 0.5 * elv + 2 * U * (mu * mu + sv * sv + np.abs(lv) + 1)
        valid = (np.arange(rows_all) < n)[:, None]
        chains.append(dict(a0=a0, h1=h1, eh1=eh1, h2=h2, eh2=eh2, mu=mu, emu=emu, lv=lv, elv=elv,
                           kl=np.where(valid, term, 0.0).sum(1), kl_e=np.where(valid, e_t, 0.0).sum(1),
                           kl_abs=np.where(valid, np.abs(term), 0.0).sum(1)))
    sched = schedule(F, grid, tiles)
    kl, kl_b = np.zeros((F, max(s for _, _, s, _ in sched) + 1)), np.zeros((F, max(s for _, _, s, _ in sched) + 1))
    for c, f, s, ts in sched:
        rows = np.concatenate([np.arange(t * TM, (t + 1) * TM) for t in ts])
        ch = chains[f]
        kl[f, s] = ch["kl"][rows].sum()
        kl_b[f, s] = ch["kl_e"][rows].sum() + gamma(len(rows) * E // 16 + 16) * ch["kl_abs"][rows].sum()
    exact = user_b == 0
    return dict(user_emb=user, user_emb_bound=C_BOUND * user_b,
                emb=np.where(exact, round_tf32(f32(user)), user), emb_bound=C_BOUND * (user_b + 2.0 ** -11 * np.abs(user)) * ~exact,
                emb16=np.where(exact, r16(user, fmt), user), emb16_bound=C_BOUND * _r16_bound(user, user_b, fmt),
                kl_part=kl, kl_part_bound=C_BOUND * kl_b, chains=chains)


def bounded_backward(img_all, chains, fdims, nfreq, act, alpha, fmt, n, eps, g, beta, inv_batch, S, grid):
    """The backward kernel's partials with bounds: {(feature, slot): {block: (value, bound)}}.  g is the S-scaled gradient
    as the kernel reads it; beta inv_batch S must be exact in fp32 (powers of two)."""
    F = len(fdims)
    tiles = -(-n // TM)
    rows_all = tiles * TM
    bs = float(f32(f32(np.float32(beta) * np.float32(inv_batch)) * np.float32(S)))
    assert bs == beta * inv_batch * S, "the bounded backward needs bs = beta inv_batch S exact"
    valid = (np.arange(rows_all) < n)[:, None]
    per = []
    for f, d in enumerate(fdims):
        ch = chains[f]
        W0p, W1, W2, _, _ = split_pack(img_all[f])
        gf = np.zeros((rows_all, E))
        gf[:n] = g[:n, f * E:(f + 1) * E]
        z = _noise_rows(eps, f, rows_all, n)
        mu, emu, lv, elv = ch["mu"], ch["emu"], ch["lv"], ch["elv"]
        sgm = np.exp(0.5 * lv)
        e_sgm = sgm * (0.5 * elv + 5 * U)
        dm = bs * mu + gf
        e_dm = bs * emu + U * np.abs(dm)
        gz = gf * z
        dl = gz * sgm * 0.5 + bs * 0.5 * np.expm1(lv)
        e_dl = (np.abs(gz) * e_sgm / 2 + 3 * U * np.abs(gz * sgm) / 2 + bs * (sgm * e_sgm + U * (sgm * sgm + 1))
                + U * np.abs(dl))
        d_ = np.where(valid, np.concatenate([dm, dl], 1), 0.0)
        e_d = np.where(valid, np.concatenate([e_dm, e_dl], 1), 0.0)
        dO, e_dO = np.where(e_d > 0, d_, r16(d_, fmt)), _r16_bound(d_, e_d, fmt)
        G2, eG2 = mm_bounded(dO, e_dO, W2.T)
        a2, ea2 = act_grad_bounded(act, ch["h2"], ch["eh2"], alpha)
        v2 = G2 * a2
        e2 = np.abs(a2) * eG2 + np.abs(G2) * ea2 + U * np.abs(v2)
        dz2, e_dz2 = np.where(e2 > 0, v2, r16(v2, fmt)), _r16_bound(v2, e2, fmt)
        G1, eG1 = mm_bounded(dz2, e_dz2, W1.T)
        a1, ea1 = act_grad_bounded(act, ch["h1"], ch["eh1"], alpha)
        v1 = G1 * a1
        e1 = np.abs(a1) * eG1 + np.abs(G1) * ea1 + U * np.abs(v1)
        dz1, e_dz1 = np.where(e1 > 0, v1, r16(v1, fmt)), _r16_bound(v1, e1, fmt)
        per.append(dict(a0=ch["a0"], h1=ch["h1"], eh1=ch["eh1"], h2=ch["h2"], eh2=ch["eh2"], dO=dO, e_dO=e_dO, dz2=dz2,
                        e_dz2=e_dz2, dz1=dz1, e_dz1=e_dz1))
    out = {}
    inv_s = 1.0 / S
    for c, f, s, ts in schedule(F, grid, tiles):
        p = per[f]
        rows = np.concatenate([np.arange(t * TM, (t + 1) * TM) for t in ts])
        a0, h1, eh1, h2, eh2, dO, e_dO, dz2, e_dz2, dz1, e_dz1 = (p[k][rows] for k in (
            "a0", "h1", "eh1", "h2", "eh2", "dO", "e_dO", "dz2", "e_dz2", "dz1", "e_dz1"))
        z0 = np.zeros_like(a0)
        w2 = mm_bounded(h2.T, eh2.T, dO, e_dO)
        b2 = mm_bounded(a0.T, z0.T, dO, e_dO)
        w1 = mm_bounded(h1.T, eh1.T, dz2, e_dz2)
        b1 = mm_bounded(a0.T, z0.T, dz2, e_dz2)
        w0p = mm_bounded(dz1.T, e_dz1.T, a0)
        w_in = fdims[f] * nfreq
        blocks = dict(w0=(w0p[0][:, :w_in].T, w0p[1][:, :w_in].T), b0=(w0p[0][:, w_in], w0p[1][:, w_in]), w1=w1,
                      b1=(b1[0][w_in], b1[1][w_in]), w2=w2, b2=(b2[0][w_in], b2[1][w_in]))
        out[(f, s)] = {k: (np.ravel(v) * inv_s, C_BOUND * np.ravel(e) * inv_s) for k, (v, e) in blocks.items()}
    return out


def bounded_partial_table(parts, lay, split_stride, nslots, sentinel):
    """(values, bounds) of the partial rows: every written block, the sentinel (bound 0) elsewhere."""
    t = np.full((nslots, split_stride), sentinel, np.float64)
    b = np.zeros_like(t)
    for (f, s), blocks in parts.items():
        for k, (v, e) in blocks.items():
            o = int(lay[k][f])
            t[s, o:o + v.size], b[s, o:o + v.size] = v, e
    return t, b


def bounded_params(rng, fdims, nfreq, logvar_offset, density=1 / 16):
    """exact_params with a live logvar half: W2's logvar columns sparse on the grid 1/8, b2's logvar half on the grid 1/4
    (lv mostly within +-4)."""
    enc = exact_params(rng, fdims, nfreq, logvar_offset, density)
    for e in enc:
        e["W2"][:, E:] = sparse_dyadic(rng, (HID, E), 2, 8, density)
        e["b2"][E:] = dyadic(rng, E, 4, 4)
    return enc
