"""TEST INFRASTRUCTURE ONLY -- a float64 reference of the 16-bit integration kernels (csrc/dib_int16.cu: the TMA + wgmma GEMM
in FWD / DGRAD / WGRAD mode, the generic and the out = 1 output head, and the fused tail dib_int16_fwd2_kernel) that rounds
exactly where the kernels round.  Not collected by pytest (no test_ prefix).

Exactness.  An fp16 x fp16 or bf16 x bf16 product is exact in fp32.  When every operand lies on a dyadic grid and every
partial sum stays below 2^24 grid units, every sum a kernel forms is exact in any order (truncating alignment inside the
tensor core included), so the fp32 accumulator holds the exact float64 value.  Every function that claims this asserts the
24-bit fit (``fits``) on the magnitudes of the sum's terms.  What follows an exact accumulator is restated in numpy float32,
one operation per kernel operation, so its roundings are the kernel's:

  GEMM FWD epilogue (dib_int16.cu:214-216, 223)  out = r(act16(fl(acc + bias)));  leaky ReLU fl(alpha z)
  GEMM DGRAD epilogue (:217-223)                 out = r(fl(acc act'(x))), act'(x) in fp32 from the 16-bit x (exact for x on
                                                 the 1/16 grid; leaky ReLU alpha rounded to fp32)
  DGRAD column sums (:224, :227-244)             of the UNROUNDED fp32 values, rows < M only, per 128-row tile [tiles][C]:
                                                 each thread adds its rows r, r + 8 to 0, a xor-4 / 8 / 16 butterfly joins the
                                                 8 row pairs of a warp, then the 8 warps' totals (16-row blocks in order)
                                                 are added to 0 in order -- restated bit for bit by ``dgrad_colsums``
  GEMM WGRAD epilogue (:209-212)                 part[s] = fl(acc out_scale) over batch rows [s rps, min(M, (s+1) rps))
  head kernels (:698-756, :862-900)              z = out_act(h . w + b); dz = loss'(z) / out * ib * out_act'(z); dg = r(dz S
                                                 Wc^T act'(h)) with column sums of the unrounded dg; dWc = h^T dz, dbc = sum dz
  head partials (:759-809, :903-943)             row r belongs to warp gw = (r // ROWS) mod nw (rows gw ROWS + k nw ROWS),
                                                 nw = 8 nblocks, and warp gw to block gw // 8; block b writes [dWc | dbc |
                                                 colsum dg] of its rows, its loss and its accuracy.  ROWS = 4 (out <= 2), 1
                                                 (generic, out > 2), 8 (head1)
  fused tail (:455-626)                          g1 = r(act16(fl(D0 + b0))) e0; g2 = r(act16(fl(D1 + b1))) e1 (on chip);
                                                 logit = g2 . w + b; dzs = loss' ib out_act'; ds = dzs S; dg2 = r(ds w
                                                 act'(g2)); dg1 = r(fl(dg2 W1^T act'(g1))) e2 with per-tile column sums
                                                 (the DGRAD order); d emb = r(dg1 W0^T) e3, 128-column chunks; CTA b walks
                                                 tiles b, b + grid, ... (grid = min(tiles, SMs)) and writes [dW out (256) |
                                                 db out (1) | column sums of dg2 (256)], its loss and its accuracy.

r() is ``fp_exact.round_to``: half to even, saturating (cvt.rn.satfinite), exact subnormals.

Inexact points carry a per-element bound instead (``*_bound`` arrays; zero where the value is exact):
  * the SFU activations of dib_act16: tanh.approx.f32 (PTX ISA: maximum relative error 2^-10.987), sigmoid
    __fdividef(1, 1 + __expf(-z)) and elu __expf(z) - 1.  __expf is ex2.approx of fl(z log2 e): 2^-22 relative plus the
    rounding of the product, |z| 2^-24 relative in the result.  The bound of the 16-bit output is that error plus one
    16-bit ulp of the result.
  * the libm losses of the heads: tests/elementwise_reference.loss gives d loss / d z, the loss and the accuracy with their
    bounds, evaluated on the kernel's own z (user_pred).  Everything after it carries a first-order propagated bound (C_BOUND
    = 2 times the sum of the terms' errors plus gamma_m sum |terms| for each m-term fp32 sum), and a 16-bit output one
    16-bit ulp on top wherever its bound is not zero (a rounding that the fp32 error may move across a tie).
Every function returns float64 arrays."""
from __future__ import annotations

import numpy as np

from tests import elementwise_reference as ER
from tests.fp_exact import C_BOUND, U, act_grad, act_grad32, exact_matmul, f32, fits, gamma, quantum, r16, ulp16

ACTS = ER.ACTS
TANH_APPROX_REL = 2.0 ** -10.987
EX2_APPROX_REL = 2.0 ** -22
HEAD_WARPS = 8
F2N = 256


# ---- activations --------------------------------------------------------------------------------------------------------
def act16(act, z32, alpha, fmt):
    """r(dib_act16(act, z)) of the fp32 pre-activation z32 (float32 array) and its bound.  linear / relu / leaky ReLU are
    restated in fp32 (bound 0); tanh / sigmoid / elu are the float64 function with the SFU error plus one 16-bit ulp."""
    z = z32.astype(np.float64)
    if act == "linear":
        return r16(z, fmt), np.zeros_like(z)
    if act == "relu":
        return r16(np.maximum(z, 0.0), fmt), np.zeros_like(z)
    if act == "leaky_relu":
        v = np.where(z32 > 0, z32, np.float32(alpha) * z32).astype(np.float64)
        return r16(v, fmt), np.zeros_like(z)
    e_exp = EX2_APPROX_REL + np.abs(z) * U * 2.0
    if act == "tanh":
        v = np.tanh(z)
        e = TANH_APPROX_REL * np.abs(v)
    elif act == "sigmoid":
        v = 1.0 / (1.0 + np.exp(-z))
        e = v * (1.0 - v) * e_exp + 2.0 ** -21 * v
    elif act == "elu":
        v = np.where(z > 0, z, np.expm1(np.minimum(z, 0.0)))
        e = np.where(z > 0, 0.0, np.exp(np.minimum(z, 0.0)) * e_exp + U)
    else:
        raise ValueError(act)
    return v, e + ulp16(np.abs(v) + e, fmt)


# ---- GEMM ---------------------------------------------------------------------------------------------------------------
def gemm_fwd(a, w, b, act, alpha, fmt):
    """FWD: r(act16(fl(a w + b))) of a [M, K], w [K, N], b [N] (16-bit values, fp32 bias) -> (out, bound)."""
    acc = exact_matmul(a, w, "FWD accumulator")
    z32 = f32(acc) + f32(b)[None, :]                                     # :215 one fp32 add
    return act16(act, z32, alpha, fmt)


def dgrad_values(dz, w, x, act, alpha):
    """DGRAD's unrounded fp32 values fl(dz w^T act'(x)) (float32 [M, K]); x None: no act'."""
    acc = f32(exact_matmul(dz, np.asarray(w, np.float64).T, "DGRAD accumulator"))
    if x is None:
        return acc
    return acc * act_grad32(act, x, alpha)                               # :220 one fp32 product


def dgrad_colsums(v32):
    """The DGRAD epilogue's per-tile column sums of v32 [M, C] (rows < M), restated in its fp32 order (:224, :231, :242)."""
    M, C = v32.shape
    tiles = -(-M // 128)
    p = np.zeros((tiles * 128, C), np.float32)
    p[:M] = v32
    # row of tile = 16 w + 8 h + l  (warp w: 64 (w >> 2) + 16 (w & 3) = 16 w; lane row l = lane >> 2)
    p = p.reshape(tiles, 8, 2, 8, C)
    cs = (np.float32(0) + p[:, :, 0]) + p[:, :, 1]                       # [tiles, w, l, C]
    t1 = cs[:, :, 0::2] + cs[:, :, 1::2]                                 # xor 4: l, l ^ 1
    t2 = t1[:, :, 0::2] + t1[:, :, 1::2]                                 # xor 8: l, l ^ 2
    wt = t2[:, :, 0] + t2[:, :, 1]                                       # xor 16: l, l ^ 4
    s = np.zeros((tiles, C), np.float32)
    for w_ in range(8):                                                  # :242, warps in order
        s = s + wt[:, w_]
    return s.astype(np.float64)


def gemm_dgrad(dz, w, x, act, alpha, fmt):
    """DGRAD of dz [M, N] through w [K, N] and the activation output x [M, K] (or None) -> (out [M, K], colsums
    [ceil(M / 128), K])."""
    v = dgrad_values(dz, w, x, act, alpha)
    return r16(v.astype(np.float64), fmt), dgrad_colsums(v)


def gemm_wgrad(g, dz, M, nsplit, rps, out_scale):
    """WGRAD split partials [nsplit, K, N] of out_scale g^T dz over batch rows [s rps, min(M, (s + 1) rps))."""
    g, dz = np.asarray(g, np.float64), np.asarray(dz, np.float64)
    out = np.zeros((nsplit, g.shape[1], dz.shape[1]))
    for s in range(nsplit):
        lo, hi = s * rps, min(M, (s + 1) * rps)
        if hi > lo:
            acc = exact_matmul(g[lo:hi].T, dz[lo:hi], "WGRAD accumulator")
            out[s] = (f32(acc) * np.float32(out_scale)).astype(np.float64)   # :212
    return out


# ---- output heads -------------------------------------------------------------------------------------------------------
def head_rows_per_warp(out_dim, head1):
    return 8 if head1 else (4 if out_dim <= 2 else 1)


def head_block_of_rows(n, nblocks, out_dim, head1):
    """The block each row is credited to (:679, :839): warp gw takes rows gw ROWS + k nw ROWS + [0, ROWS)."""
    rows = head_rows_per_warp(out_dim, head1)
    nw = HEAD_WARPS * nblocks
    return ((np.arange(n) // rows) % nw) // HEAD_WARPS


def _loss_rows(loss, out_act, alpha, z, zb, y, ib, w, exact):
    """The row loss, accuracy and dz of the compiled loss on the output z; exact (MSE, linear output, power-of-two 1 / out
    and inv_batch, dyadic operands): float64 values with zero bounds, else tests/elementwise_reference.loss on z."""
    n, C = z.shape
    if exact:
        t = np.asarray(y, np.float64).reshape(n, C)
        wv = np.ones(n) if w is None else np.asarray(w, np.float64)
        d = z - t
        l = (d * d * wv[:, None]).sum(-1) / C
        acc = ((z > 0.5).astype(np.float64) == t).sum(-1) / C
        dz = 2.0 * d / C * (ib * wv)[:, None]
        fits(np.abs(d * d * wv[:, None]).sum(-1), quantum(d) ** 2 * quantum(wv), "row loss")
        fits(np.abs(dz), quantum(dz), "dz")
        zero = np.zeros(n)
        return dict(row_loss=l, row_loss_bound=zero, row_acc=acc, row_acc_bound=zero, dz=dz, dz_bound=np.zeros_like(dz))
    r = ER.loss(loss, out_act, alpha, z, y, ib, w)
    # the z the kernel computed carries its own bound: it moves dz by at most |d dz / d z| zb, here bounded by the loss's
    # curvature times zb (every loss here has |d^2 l / d z^2| <= 2 / out_dim on the scale of ib, except BCE on
    # probabilities, whose curvature 1 / p^2 is taken at the clipped z)
    if np.any(zb > 0):
        if loss == "bce_probs":
            pc = np.clip(z, ER.KERAS_EPS, ER.ONE_M_EPS)
            curv = 1.0 / np.minimum(pc, 1.0 - pc) ** 2
        else:
            curv = 2.0 * np.ones_like(z)
        wv = np.ones(n) if w is None else np.asarray(w, np.float64)
        r["dz_bound"] = r["dz_bound"] + C_BOUND * curv * zb / C * (ib * wv)[:, None]
    return r


def head(g, Wc, bc, out_act, hid_act, alpha, loss, y, ib, S, w=None, nblocks=1, head1=False, fmt="fp16", z_kernel=None,
         train=True, exact=False):
    """The output head over g [n, K] (16-bit values), Wc [K, out], bc [out] (fp32).  Returns z [n, out] (+ bound), and with
    y: per-row loss / accuracy, per-block loss_part / acc_part [nblocks]; in training dg [n, K] and wpart [nblocks, K out +
    out + K], each with a bound.  z_kernel: the kernel's z (user_pred), on which the loss is evaluated when not exact."""
    g, Wc, bc = (np.asarray(v, np.float64) for v in (g, Wc, bc))
    n, K = g.shape
    out = Wc.shape[1]
    logit = exact_matmul(g, Wc, "head logits") + bc[None, :] if exact else g @ Wc + bc[None, :]
    if exact:
        assert out_act == "linear"
        fits(np.abs(g) @ np.abs(Wc) + np.abs(bc), min(quantum(g) * quantum(Wc), quantum(bc)), "head logit + bias")
        z, zb = logit, np.zeros_like(logit)
    else:
        e_logit = gamma(K + 6) * (np.abs(g) @ np.abs(Wc) + np.abs(bc))
        z = logit
        if out_act == "linear":
            zb = e_logit
        elif out_act == "sigmoid":
            z = 1.0 / (1.0 + np.exp(-logit))
            zb = z * (1 - z) * e_logit + 7 * U * z
        else:
            raise ValueError("the bounded head takes a linear or sigmoid output")
        zb = C_BOUND * zb
    res = dict(z=z, z_bound=zb)
    blk = head_block_of_rows(n, nblocks, out, head1)
    if y is None:
        res.update(loss_part=np.zeros(nblocks), loss_part_bound=np.zeros(nblocks), acc_part=np.zeros(nblocks),
                   acc_part_bound=np.zeros(nblocks))
        dz, dz_b = np.zeros((n, out)), np.zeros((n, out))
    else:
        zl = z if exact or z_kernel is None else np.asarray(z_kernel, np.float64).reshape(n, out)
        lr = _loss_rows(loss, out_act, alpha, zl, 0 * zb if z_kernel is not None else zb, y, ib, w, exact)
        for key, rk in (("loss_part", "row_loss"), ("acc_part", "row_acc")):
            res[key] = np.bincount(blk, lr[rk], nblocks) + 0.0
            res[key + "_bound"] = np.bincount(blk, lr[rk + "_bound"], nblocks) + gamma(n + 8) * np.bincount(blk, np.abs(lr[rk]), nblocks)
            if exact:
                fits(np.bincount(blk, np.abs(lr[rk]), nblocks), quantum(lr[rk]), key)
                res[key + "_bound"] = np.zeros(nblocks)
        res["row_loss"], res["row_acc"] = lr["row_loss"], lr["row_acc"]
        dz, dz_b = lr["dz"], lr["dz_bound"]
    if not train:
        return res
    a = act_grad32(hid_act, g, alpha).astype(np.float64)
    # unrounded dg = (s S) act'.  head1 forms s = dz w as one product (:890-895), so a zero w keeps the sign of dz; the
    # generic kernel sums fma(dz_o, w_io, s) from +0 (:745-748), so an exactly zero s is +0 -- matmul's zeros are the same
    s_ = dz[:, :1] * Wc.T if head1 else dz @ Wc.T
    d = S * s_ * a
    if exact:
        fits(np.abs(dz) @ np.abs(Wc.T) * S, quantum(dz) * quantum(Wc) * S, "head dg sums")
        d_b = np.zeros_like(d)
        assert np.array_equal(f32(d).astype(np.float64), d), "head dg: s S act' is not exact"
    else:
        d_b = S * np.abs(a) * (dz_b @ np.abs(Wc.T) + gamma(out + 3) * (np.abs(dz) @ np.abs(Wc.T)))
    res["dg"] = r16(d, fmt)
    res["dg_bound"] = np.zeros_like(d) if exact else np.where(d_b > 0, d_b + ulp16(np.abs(d) + d_b, fmt), 0.0)
    parts = np.zeros((nblocks, K * out + out + K))
    pb = np.zeros_like(parts)
    qg, qdz, qd = (quantum(v) for v in (g, dz, d)) if exact else (1.0, 1.0, 1.0)
    for b in range(nblocks):
        rows = blk == b
        gb, dzb, db_ = g[rows], dz[rows], d[rows]
        nb = int(rows.sum())
        # + 0.0: every kernel accumulator starts at +0, so a sum of zeros is +0 whatever their signs
        parts[b, :K * out] = (gb.T @ dzb).ravel() + 0.0
        parts[b, K * out:K * out + out] = dzb.sum(0) + 0.0
        parts[b, K * out + out:] = db_.sum(0) + 0.0
        if exact:
            fits((np.abs(gb).T @ np.abs(dzb)).ravel(), qg * qdz, "head dWc")
            fits(np.abs(dzb).sum(0), qdz, "head dbc")
            fits(np.abs(db_).sum(0), qd, "head dg column sums")
        else:
            gm = gamma(nb + 8)
            pb[b, :K * out] = (np.abs(gb).T @ dz_b[rows] + gm * (np.abs(gb).T @ np.abs(dzb))).ravel()
            pb[b, K * out:K * out + out] = dz_b[rows].sum(0) + gm * np.abs(dzb).sum(0)
            pb[b, K * out + out:] = d_b[rows].sum(0) + gm * np.abs(db_).sum(0)
    res["wpart"], res["wpart_bound"] = parts, pb
    return res


# ---- the fused tail -----------------------------------------------------------------------------------------------------
def fwd2(a, W0, b0, W1, b1, wout, bout, act, alpha, y, ib, S, sms, fmt, w=None, stages=3, demb=False):
    """The fused tail in its exact regime (act in linear / relu / leaky ReLU, MSE, a linear output, dyadic operands,
    power-of-two inv_batch and S).  a [M, K0] (16-bit values), W0 [K0, 256], W1 [256, 256] (16-bit values), b0, b1, wout
    [256], bout [1] fp32.  stages: 1 = forward only, 2 = + dg2 and the partials, 3 = + dg1 / dbpart, demb: + d emb.
    Returns g1, z, loss_part, acc_part (and dg2, wpart, dg1, dbpart, demb) with grid = min(tiles, sms)."""
    assert act in ("linear", "relu", "leaky_relu"), "the exact tail needs an activation without SFU"
    a, W0, W1 = (np.asarray(v, np.float64) for v in (a, W0, W1))
    M = a.shape[0]
    g1 = act16(act, f32(exact_matmul(a, W0, "D0")) + f32(b0)[None, :], alpha, fmt)[0]            # e0 :464
    g2 = act16(act, f32(exact_matmul(g1, W1, "D1")) + f32(b1)[None, :], alpha, fmt)[0]           # e1 :483
    wout = np.asarray(wout, np.float64)
    zp = exact_matmul(g2, wout[:, None], "logit")[:, 0]
    z = (f32(zp) + np.float32(bout[0])).astype(np.float64)               # :502 (linear output)
    fits(np.abs(zp) + abs(bout[0]), min(quantum(zp), quantum(bout)), "logit + bias")
    tiles = -(-M // 128)
    grid = min(tiles, sms)
    cta = (np.arange(M) // 128) % grid                                   # tile t runs on CTA t mod grid
    res = dict(g1=g1, z=z, grid=grid)
    if y is not None:
        lr = _loss_rows("mse", "linear", alpha, z[:, None], np.zeros((M, 1)), y, ib, w, True)
        res["loss_part"] = np.bincount(cta, lr["row_loss"], grid)
        res["acc_part"] = np.bincount(cta, lr["row_acc"], grid)
        fits(np.bincount(cta, np.abs(lr["row_loss"]), grid), quantum(lr["row_loss"]), "tail loss sums")
        dzs = lr["dz"][:, 0]
    else:
        res["loss_part"], res["acc_part"] = np.zeros(grid), np.zeros(grid)
        dzs = np.zeros(M)
    if stages < 2:
        return res
    ds = dzs * S
    d2 = ds[:, None] * wout[None, :] * act_grad32(act, g2, alpha).astype(np.float64)          # e1 pass 3 :551
    fits(np.abs(d2), quantum(d2), "dg2")
    res["dg2"] = r16(d2, fmt)
    wp = np.zeros((grid, 2 * F2N + 1))
    qg2, qdzs, qd2 = quantum(g2), quantum(dzs), quantum(d2)
    for b in range(grid):
        rows = cta == b
        wp[b, :F2N] = g2[rows].T @ dzs[rows] + 0.0                                              # pass 2 :532
        wp[b, F2N] = dzs[rows].sum() + 0.0                                                      # (+ 0.0: sums start at +0)
        wp[b, F2N + 1:] = d2[rows].sum(0) + 0.0                                                 # pass 3 :552 (unrounded)
        fits(np.abs(g2[rows]).T @ np.abs(dzs[rows]), qg2 * qdzs, "dW out")
        fits(np.abs(dzs[rows]).sum(), qdzs, "db out")
        fits(np.abs(d2[rows]).sum(0), qd2, "dg2 column sums")
    res["wpart"] = wp
    if stages < 3:
        return res
    v1 = dgrad_values(res["dg2"], W1, g1, act, alpha)                    # e2 :585-590
    res["dg1"] = r16(v1.astype(np.float64), fmt)
    res["dbpart"] = dgrad_colsums(v1)
    if demb:
        res["demb"] = r16(exact_matmul(res["dg1"], W0.T, "d emb"), fmt)  # e3 :620
    return res


def _act_value_grad(act, h):
    """dib_act_grad(act, h) in float64 from the float64 output h (the SFU activations: all smooth, |d act' / dh| <= 2)."""
    if act == "tanh":
        return 1.0 - h * h
    if act == "sigmoid":
        return h * (1.0 - h)
    if act == "elu":
        return np.where(h > 0, 1.0, h + 1.0)
    raise ValueError(act)


def tc_gamma(k):
    """The error factor of a k-term fp32 sum inside the tensor core, whose alignment may truncate: 2u per add."""
    return gamma(2 * k)


def fwd2_sfu(a, W0, b0, W1, b1, wout, bout, act, alpha, y, ib, S, sms, fmt, kern, w=None, stages=3, demb=False):
    """The fused tail with an SFU activation (tanh / sigmoid / elu), MSE and a linear output, each output with a bound.
    g1 is bounded from the exact D0 by the SFU error plus one 16-bit ulp (act16).  Every later stage continues from the
    kernel's own stored intermediates in ``kern`` (float64 values): D1 from kern['g1'], the loss and d loss / d logit from
    kern['z'] (user_pred, through tests/elementwise_reference.loss), dg1 from kern['dg2'], d emb from kern['dg1'].  Only g2,
    which never leaves the chip, carries a propagated bound into the logit, dg2 and the partials.  Sums inside the tensor
    core are charged tc_gamma, fp32 sums gamma, and every propagated bound is C_BOUND times its first-order terms; a 16-bit
    output gets one 16-bit ulp on top."""
    assert act in ("tanh", "sigmoid", "elu")
    a, W0, W1, wout = (np.asarray(v, np.float64) for v in (a, W0, W1, wout))
    M, C = a.shape[0], C_BOUND
    ulp = lambda v, e: e + ulp16(np.abs(v) + e, fmt)
    g1, g1_b = act16(act, f32(exact_matmul(a, W0, "D0")) + f32(b0)[None, :], alpha, fmt)        # e0 :464
    g1k = np.asarray(kern["g1"], np.float64)
    d1 = g1k @ W1
    z1 = d1 + f32(b1)[None, :].astype(np.float64)
    e_z1 = tc_gamma(F2N) * (np.abs(g1k) @ np.abs(W1)) + U * np.abs(z1)
    g2, e_sfu = act16(act, f32(z1), alpha, fmt)                                                   # e1 :483, on chip
    e_g2 = e_z1 + e_sfu                                     # |act'| <= 1; e_sfu holds the SFU error and the 16-bit ulp
    zp = g2 @ wout
    z = zp + float(np.float32(bout[0]))                                                           # :491, :502
    e_z = e_g2 @ np.abs(wout) + gamma(F2N + 8) * (np.abs(g2) @ np.abs(wout)) + U * np.abs(z)
    tiles = -(-M // 128)
    grid = min(tiles, sms)
    cta = (np.arange(M) // 128) % grid
    res = dict(g1=g1, g1_bound=g1_b, z=z, z_bound=C * e_z, grid=grid)
    zk = np.asarray(kern["z"], np.float64)
    if y is not None:
        lr = ER.loss("mse", "linear", alpha, zk[:, None], y, ib, w)
        n_cta = np.bincount(cta, minlength=grid)
        for key, rk in (("loss_part", "row_loss"), ("acc_part", "row_acc")):
            res[key] = np.bincount(cta, lr[rk], grid)
            res[key + "_bound"] = np.bincount(cta, lr[rk + "_bound"], grid) + C * gamma(n_cta + 40) * np.bincount(cta, np.abs(lr[rk]), grid)
        dzs, e_dzs = lr["dz"][:, 0], lr["dz_bound"][:, 0]
    else:
        z0 = np.zeros(grid)
        res.update(loss_part=z0, loss_part_bound=z0, acc_part=z0, acc_part_bound=z0)
        dzs, e_dzs = np.zeros(M), np.zeros(M)
    if stages < 2:
        return res
    ap = _act_value_grad(act, g2)
    e_ap = 2.0 * e_g2 + 2 * U * np.abs(ap)
    ds = dzs * S
    d2 = ds[:, None] * wout[None, :] * ap                                                         # e1 pass 3 :551
    e_d2 = np.abs(wout)[None, :] * (np.abs(ap) * S * e_dzs[:, None] + np.abs(ds)[:, None] * e_ap) + 3 * U * np.abs(d2)
    res["dg2"], res["dg2_bound"] = r16(d2, fmt), ulp(d2, C * e_d2)
    wp, wb = np.zeros((grid, 2 * F2N + 1)), np.zeros((grid, 2 * F2N + 1))
    for b in range(grid):
        rows = cta == b
        gm = gamma(int(rows.sum()) + 16)
        wp[b, :F2N] = g2[rows].T @ dzs[rows]                                                      # pass 2 :532
        wb[b, :F2N] = (e_g2[rows].T @ np.abs(dzs[rows]) + np.abs(g2[rows]).T @ e_dzs[rows]
                       + gm * (np.abs(g2[rows]).T @ np.abs(dzs[rows])))
        wp[b, F2N] = dzs[rows].sum()
        wb[b, F2N] = e_dzs[rows].sum() + gm * np.abs(dzs[rows]).sum()
        wp[b, F2N + 1:] = d2[rows].sum(0)                                                         # pass 3 :552 (unrounded)
        wb[b, F2N + 1:] = e_d2[rows].sum(0) + gm * np.abs(d2[rows]).sum(0)
    res["wpart"], res["wpart_bound"] = wp, C * wb
    if stages < 3:
        return res
    dg2k = np.asarray(kern["dg2"], np.float64)
    acc2 = dg2k @ W1.T                                                                            # D1 :574
    e_acc2 = tc_gamma(F2N) * (np.abs(dg2k) @ np.abs(W1.T))
    a1, e_a1 = act_grad(act, np.asarray(kern["g1"], np.float64), alpha)
    v1 = acc2 * a1                                                                                # e2 :585
    e_v1 = np.abs(a1) * e_acc2 + np.abs(acc2) * e_a1 + U * np.abs(v1)
    res["dg1"], res["dg1_bound"] = r16(v1, fmt), ulp(v1, C * e_v1)
    pad = tiles * 128 - M
    tile_sum = lambda x: np.pad(x, ((0, pad), (0, 0))).reshape(tiles, 128, -1).sum(1)
    res["dbpart"] = tile_sum(v1)
    res["dbpart_bound"] = C * (tile_sum(e_v1) + gamma(128 + 8) * tile_sum(np.abs(v1)))
    if demb:
        dg1k = np.asarray(kern["dg1"], np.float64)
        acc = dg1k @ W0.T                                                                         # D0, e3 :613-620
        res["demb"] = r16(acc, fmt)
        res["demb_bound"] = ulp(acc, C * tc_gamma(F2N) * (np.abs(dg1k) @ np.abs(W0.T)))
    return res
