"""TEST INFRASTRUCTURE ONLY -- a float64 reference of the elementwise kernels of the training step (csrc/dib_elementwise.cu:
the reparameterisation forward and backward with the per-feature KL, the compiled loss with its accuracy and d loss / d z,
the positional encoding, dropout, and the fixed-order reductions) with a worst-case error bound next to every output,
derived from the fp32 arithmetic the kernels do.

Values.  Every output is computed in float64 from the kernels' fp32 inputs with formulas that do not cancel: the KL term
mu^2 + (e^lv - 1 - lv) takes expm1 and, below |lv| = 0.01, its Taylor series; the softmax cross-entropy is logsumexp - z_label.

Bounds (running error analysis).  u = 2^-24, gamma_m = m u / (1 - m u).  Each kernel statement is restated below, in the
kernel's order of operations, on a pair (value, e): e bounds the distance of the kernel's fp32 value from the exact one.
An fp32 operation with exact result r adds u |r| (round to nearest); its operands' errors propagate to first order through
its derivative (a product keeps the e_a e_b term).  The libm routines the kernels call (the library is built without
fast-math): expf 2 ulp (4u |r|), logf / log1pf / expm1f 1 ulp (2u |r|), sinf 2 ulp; an fp32 constant such as 0.16666667 is
exact as stored.  fmaf and a compiler-contracted a * b + c round once, so charging both roundings only widens the bound.
The bound reported is C = C_BOUND = 2 times e: the factor covers every product of two or more rounding errors (every
first-order term here is far below 1e-2).  Every sum is bounded by its terms: a serial chain of m adds by gamma_m sum |terms|
plus the terms' own errors, never by the size of its result, so sums that cancel are covered.

  reparam_fwd (dib_reparam_fwd_kernel), per (row, feature f, e):
      s = expf(0.5 lv): 4u s;   u = fmaf(s, z, mu): |z| 4u s + s e_z + u |u|
      z is eps (exact) or the Philox normal; the kernel's Box-Muller runs on the SFU approximations (lg2 / sin / cos .approx,
      dib_common.cuh), whose error bounds PTX states loosely, so e_z against oracle/philox.normal_noise (libm, float64) is set
      from measurement: Z_TOL (1 + |z|), Z_TOL = 2^-15.  The kernel's own noise (mu = lv = 0 makes u = z exactly) measures
      at most 0.11 of it on an H100 (tests/test_gpu_elementwise_kernels.py::test_philox_noise_against_normal_noise checks it
      without the factor C), so C keeps its meaning for the other terms.
      KL term k = 0.5 dib_kl_term(mu, lv): for |lv| < 1/16 the series lv^2 (1/2 + lv (1/6 + lv (1/24 + lv / 120))), five
      products and three adds, each within 1.07 |its value| of the final r: 10u r, plus the dropped tail lv^6 / 720 (1 + |lv|);
      else expm1f(lv) - lv: 2u |expm1 lv| + u |r|.  Then fmaf(mu, mu, r): u |mu^2 + r|; the factor 0.5 is exact.
      emb = u (TF32-rounded under round_out: plus half a TF32 ulp, 2^-11 (|u| + bound));  user_emb = u unrounded.
      kl_part[f, b]: each thread adds its E terms in order, then a 5-level shuffle tree and 8 warp sums in order:
      gamma_{E + 13} sum |k| + sum e_k.  Padding rows of padded sets give exactly 0 (u, KL and their gradient).
  reparam_bwd (dib_reparam_bwd_kernel): bs = fl(beta inv_batch): u |bs|;
      d mu = fmaf(bs, mu, du):  |mu| u |bs| + u |d mu|
      d lv = fmaf(fl(du z), fl(0.5 s), fl(fl(bs 0.5) expm1f(lv))):
             |du| e_z |s| / 2 + |du z s / 2| (u + 4u) + |c| (u + 2u + u) + u |d lv|,  c = bs expm1(lv) / 2.
  loss (dib_loss_kernel), one row per thread.  The output activation's derivative a' comes from the output h (dib_act_grad):
      exact for linear / relu / leaky relu; tanh 1 - h h: u h^2 + u |1 - h^2|; sigmoid h (1 - h): u |h (1 - h)| 2 (two
      roundings); elu h + 1: u |h + 1|.
      sparse CE: m = max z (exact), e_j = expf(fl(z_j - m)): e_j (u |z_j - m| + 4u); se = sum_j e_j in order:
        e_se = gamma_C sum e_j + sum e_ej; logf(se): e_se / se + 2u |log se|; l = fl(fl(m + log se) - z_label): + u |m + log se|
        + u |l|; weighted: fl(l w): + u |l w|.  p_j = fl(e_j fl(1 / se)): p_j (rel(e_j) + e_se / se + 2u);
        g_j = fl(p_j - [j = label]): + u |g_j|;  dz_j = fl(fl(g_j ib) a'): |ib a'| e_g + |g ib| e_a' + 2u |dz|,
        ib = inv_batch (weighted: fl(inv_batch w), + u).
        A label outside (-1, C), NaN included, gives NaN loss, NaN dz for the whole row and accuracy 0 (dib_sparse_label).
      per-output losses (dib_loss_add / dib_loss_add_w), summed in order over the outputs and scaled by fl(1 / out):
        BCE on logits: max(z, 0) - z t + log1pf(expf(-|z|)): u |z t| + (4u + 2u) L1 + 3 u-roundings of the partial results,
          L1 = log1p(e^-|z|);  g = fl(fl(1 / fl(1 + expf(-z))) - t): sigma (4u + 2u) + u |g|  (expf(-z) e^-z 4u relative);
          below z = -88.7 expf(-z) overflows and sigma comes out 0: + sigma where sigma < 2^-126.
        BCE on probabilities: p~ = clip(z, eps, 1 - eps) (exact); each logf(fl(p~ + eps)) 2u |log| + u (p~ + eps) / (p~ + eps),
          times t and 1 - t, summed: 3 roundings;  g = -t / (p~ + eps) + (1 - t) / (1 - p~ + eps): 4u |each term| + u |g|.
        MSE: d = fl(z - t): u |d|;  l += d d: 2 |d| u |d| + u |d^2|;  g = 2 d: 2u |d|.
        The row loss sums out_dim terms in order: gamma_out sum |terms| + sum e; then times fl(1 / out): + 2u |l|.
        dz_j = fl(fl(fl(g inv_out) ib) a'): like sparse CE plus 2u |g inv_out| for inv_out.
      accuracy: sparse CE (float)argmax == t, exact; per-output (z > 0.5) == t, a count times fl(1 / out): exact when out is
        a power of two, else within 2u |acc|.
      loss_part / acc_part: 256-row blocks summed by a 5-level shuffle tree and 8 warp sums in order: gamma_13 sum |rows| +
        sum e_rows; exact for the accuracy count when every row's accuracy is exact.
      A result that is subnormal or underflows adds up to SUB = 2^-149 per operation on top (|z| up to 88 reaches them).
  pe (dib_pe_kernel): f = 0 copies x (exact); else sinf(fl(f x)): |cos(f x)| u |f x| + 4u |sin(f x)| + TINY.
  dropout (dib_dropout_kernel): fl(x keep) with keep = fl(1 / (1 - rate)) on the kept columns, 0 on the dropped ones: one
      fp32 product, restated exactly in numpy float32 (bit for bit).
  reductions (reduce_partials, reduce_segments, finalize_stats): the tests feed integer-valued operands whose partial sums are
      all below 2^24, and powers of two as scales, so every summation order gives the same exact result (bit for bit).

  pe_plain (dib_pe_plain_kernel, dib_positional_encoding): block 0 copies x; block k: sinf(2^k x), 2^k x exact:
      4u |sin| + u |cos| |2^k x| + TINY (the u |2^k x| covers sinf's argument reduction relative to the exact argument).
  adam (dib_adam_kernel), t = step + 1: lr_t = fl(fl(lr (float)sqrt(1 - b2^t)) / (float)(1 - b1^t)) (double inside):
      4u |lr_t|;  c1 = 1 - b1, c2 = 1 - b2 exact (Sterbenz, b in [1/2, 1]);  m' = m + fl(g - m) c1: 2u |c1 (g - m)| + u |m'|;
      v' = v + fl(g^2 - v) c2: c2 (u g^2 + u |g^2 - v|) + u |c2 (g^2 - v)| + u |v'|;  sq = sqrtf(v'): min(e_v' / 2 sq,
      sqrt(e_v')) + u sq;  w' = w - fl(fl(lr_t m') / fl(sq + eps)): (|m'| e_lr + lr_t e_m' + u |lr_t m'| + |q| (e_sq + u den))
      / den + u |q| + u |w'|; g^2 and the moments can be subnormal (g = 1e-20): + SUB per such product.
  sgd (dib_sgd_kernel): momentum 0: w - fl(lr g): u |lr g| + u |w'|;  else v' = fl(fl(mom v) - fl(lr g)): u (|mom v| +
      |lr g| + |v'|); w' = w + v' or, Nesterov, w + fl(fl(mom v') - fl(lr g)): mom e_v' + u (|mom v'| + |lr g| + |inner|),
      + u |w'|.
  rmsprop (dib_rmsprop_kernel): ms' = fl(fl(rho ms) + fl(c g^2)), c = 1 - rho exact: u (|rho ms| + 2 c g^2 + |ms'|);
      den = sqrtf(fl(ms' + eps)): (e_ms' + u (ms' + eps)) / (2 den) + u den;  t = fl(fl(lr g) / den): (u |lr g| + |t| e_den)
      / den + u |t|;  mom' = fl(fl(momentum mom) + t): u |momentum mom| + e_t + u |mom'|;  w' = fl(w - mom'): + u |w'|.
  pairwise (dib_pairwise_gauss_kernel), the values cancellation-free: log sbar - (la + lb) / 2 = log cosh((la - lb) / 2) and
      lb - la - 1 + e^(la - lb) = expm1(la - lb) - (la - lb).  Every sum over e, in whatever order the compiler groups it,
      is bounded by gamma_N sum |subterms| (N = the number of subterms) plus the subterms' own errors:
      kind 0: t1 = sum d^2 / sbar (sbar = 0.5 fl(expf(la) + expf(lb)), relative 5u; d^2 / sbar: 6u + 2u + its relative
      error), t2 = sum (logf(sbar) - 0.5 fl(la + lb)) with logf 5u / 1 + 2u |log sbar|; D = 0.125 t1 + 0.5 t2: + u |D|;
      kind 1: D = 0.5 sum ((lb - la) - 1 + expf(la - lb) + d^2 expf(-lb)), expf(la - lb): (4u + u |la - lb|) e^(la - lb),
      d^2 e^-lb: 8u of it;  exp(-D): e^-D (e_D + 4u) + TINY.

round_out is cvt.rna.tf32.f32 applied to an output.
Every function returns float64 arrays.  The product path never imports this."""
from __future__ import annotations

import numpy as np

from tests.fp_exact import C_BOUND, TINY, U, act_grad, gamma

SUB = 2.0 ** -149            # an operation whose result is subnormal or underflows: up to one subnormal step absolutely
Z_TOL = 2.0 ** -15
TF32_HALF_ULP = 2.0 ** -11
ACTS = ("linear", "relu", "tanh", "leaky_relu", "sigmoid", "elu")
LOSSES = {"bce_logits": 0, "sparse_ce_logits": 1, "mse": 2, "external": 3, "bce_probs": 4}
KERAS_EPS = float(np.float32(1e-7))
ONE_M_EPS = float(np.float32(1.0) - np.float32(1e-7))
ROWS_PER_BLOCK = 256


def f64(a):
    return np.asarray(a, np.float64)


def sparse_label(t, C):
    """dib_sparse_label: (int)t for -1 < t < C, else -1 (NaN included)"""
    t = f64(t)
    ok = (t > -1.0) & (t < C)
    return np.where(ok, np.trunc(np.where(ok, t, 0.0)), -1).astype(np.int64)


# ---- reparameterisation -------------------------------------------------------------------------------------------------
def kl_r(lv):
    """e^lv - 1 - lv in float64 without cancellation"""
    lv = f64(lv)
    series = lv * lv * (0.5 + lv * (1 / 6 + lv * (1 / 24 + lv * (1 / 120 + lv * (1 / 720 + lv / 5040)))))
    return np.where(np.abs(lv) < 0.01, series, np.expm1(lv) - lv)


def kl_term_bound(mu, lv):
    """the error bound of one kernel KL term k = 0.5 dib_kl_term(mu, lv) (before C_BOUND)"""
    mu, lv = f64(mu), f64(lv)
    r = kl_r(lv)
    small = np.abs(lv) < 0.0625
    e_r = np.where(small, 10 * U * r + lv ** 6 / 720 * (1 + np.abs(lv)), 2 * U * np.abs(np.expm1(lv)) + U * np.abs(r))
    return 0.5 * (e_r + U * np.abs(mu * mu + r))


def reparam_forward(mu, lv, z, z_tol=0.0, real=None):
    """mu, lv, z [F, n, E] (fp32 values; z the noise, exact when z_tol = 0, else the float64 Philox normal) and real [n] (None:
    every row) -> u, u_bound [F, n, E], kl [F, n, E] (the per-element 0.5 (mu^2 + e^lv - 1 - lv)), kl_part, kl_part_bound
    [F, ceil(n / 256)]."""
    mu, lv, z = f64(mu), f64(lv), f64(z)
    F, n, E = mu.shape
    s = np.exp(0.5 * lv)
    u = mu + s * z
    e_z = z_tol * (1.0 + np.abs(z))
    u_b = np.abs(z) * 4 * U * s + s * e_z + U * np.abs(u)
    kl = 0.5 * (mu * mu + kl_r(lv))
    kl_b = kl_term_bound(mu, lv)
    if real is not None:
        m = np.asarray(real, bool)[None, :, None]
        u, u_b, kl, kl_b = (np.where(m, a, 0.0) for a in (u, u_b, kl, kl_b))
    nblk = -(-n // ROWS_PER_BLOCK)
    pad = nblk * ROWS_PER_BLOCK - n
    kr = np.pad(kl.sum(-1), ((0, 0), (0, pad))).reshape(F, nblk, ROWS_PER_BLOCK)
    kb = np.pad(kl_b.sum(-1), ((0, 0), (0, pad))).reshape(F, nblk, ROWS_PER_BLOCK)
    part = kr.sum(-1)
    part_b = gamma(E + 13) * np.abs(kr).sum(-1) + kb.sum(-1)
    return dict(u=u, u_bound=C_BOUND * u_b, kl=kl, kl_bound=C_BOUND * kl_b, kl_part=part, kl_part_bound=C_BOUND * part_b)


def reparam_backward(mu, lv, z, du, beta, inv_batch, z_tol=0.0, real=None):
    """d mu, d lv [F, n, E] from du [F, n, E] (the gradient at u), beta and inv_batch (fp32 values), with bounds."""
    mu, lv, z, du = f64(mu), f64(lv), f64(z), f64(du)
    bs = float(np.float32(beta)) * float(np.float32(inv_batch))
    e_bs = U * abs(bs)
    s = np.exp(0.5 * lv)
    em1 = np.expm1(lv)
    dmu = du + bs * mu
    dmu_b = np.abs(mu) * e_bs + U * np.abs(dmu)
    c = bs * 0.5 * em1
    dlv = du * z * 0.5 * s + c
    e_z = z_tol * (1.0 + np.abs(z))
    dlv_b = (np.abs(du) * e_z * 0.5 * s + np.abs(du * z * 0.5 * s) * 5 * U + np.abs(c) * 4 * U + 0.5 * np.abs(em1) * e_bs
             + U * np.abs(dlv))
    if real is not None:
        m = np.asarray(real, bool)[None, :, None]
        dmu, dmu_b, dlv, dlv_b = (np.where(m, a, 0.0) for a in (dmu, dmu_b, dlv, dlv_b))
    return dict(dmu=dmu, dmu_bound=C_BOUND * dmu_b, dlv=dlv, dlv_bound=C_BOUND * dlv_b)


def kl_term_old_fp32(mu, lv):
    """the KL term as the kernels formed it before dib_kl_term, in fp32: 0.5f * (mu*mu + expf(lv) - lv - 1.f)"""
    mu, lv = np.asarray(mu, np.float32), np.asarray(lv, np.float32)
    one, half = np.float32(1.0), np.float32(0.5)
    return (half * (((mu * mu + np.exp(lv)) - lv) - one)).astype(np.float64)


def kl_term_fp32(mu, lv):
    """dib_kl_term(mu, lv) / 2 restated in numpy fp32 (expm1 rounded once to fp32, as a 1-ulp expm1f may)"""
    mu, lv = np.asarray(mu, np.float32), np.asarray(lv, np.float32)
    c = [np.float32(v) for v in (0.5, 0.16666667, 0.041666668, 0.008333334)]
    series = lv * lv * (c[0] + lv * (c[1] + lv * (c[2] + lv * c[3])))
    em1 = np.expm1(lv.astype(np.float64)).astype(np.float32)
    r = np.where(np.abs(lv) < np.float32(0.0625), series, em1 - lv)
    return (np.float32(0.5) * (mu.astype(np.float64) * mu + r).astype(np.float32)).astype(np.float64)


# ---- loss -------------------------------------------------------------------------------------------------------------
def _block_sums(rows, rows_b, n):
    nblk = -(-n // ROWS_PER_BLOCK)
    pad = nblk * ROWS_PER_BLOCK - n
    r = np.pad(rows, (0, pad)).reshape(nblk, ROWS_PER_BLOCK)
    b = np.pad(rows_b, (0, pad)).reshape(nblk, ROWS_PER_BLOCK)
    return r.sum(-1), gamma(13) * np.abs(r).sum(-1) + b.sum(-1)


def loss(kind, act, alpha, z, y, inv_batch, w=None):
    """The compiled loss of rows z [n, out] (the output activation's OUTPUT, fp32 values) against y (sparse CE: [n] labels,
    external: [n, out] d task loss / d z, else [n, out]), fp32 inv_batch, optional weights w [n].  Returns row_loss, row_acc,
    dz [n, out], loss_part, acc_part [ceil(n / 256)], each with a bound (acc_bound zero where exact)."""
    z = f64(z)
    n, C = z.shape
    ib0 = float(np.float32(inv_batch))
    ib = ib0 * (f64(w) if w is not None else np.ones(n))
    e_ib = U * np.abs(ib) if w is not None else np.zeros(n)
    a, e_a = act_grad(act, z, alpha)
    wv = f64(w) if w is not None else np.ones(n)
    if kind == "external":
        g = f64(y)
        dz = g * a
        dz_b = np.abs(g) * e_a + U * np.abs(dz) + SUB
        zeros = np.zeros(n)
        lp, lpb = _block_sums(zeros, zeros, n)
        return dict(row_loss=zeros, row_loss_bound=zeros, row_acc=zeros, row_acc_bound=zeros, dz=dz, dz_bound=C_BOUND * dz_b,
                    loss_part=lp, loss_part_bound=lpb, acc_part=lp, acc_part_bound=lpb)
    if kind == "sparse_ce_logits":
        t = f64(y).reshape(n)
        lab = sparse_label(t, C)
        bad = lab < 0
        m = z.max(-1, keepdims=True)
        ex = np.exp(z - m)
        se = ex.sum(-1, keepdims=True)
        lse = m + np.log(se)
        zl = z[np.arange(n), np.maximum(lab, 0)]
        l = lse[:, 0] - zl
        rel_e = U * np.abs(z - m) + 4 * U
        e_se = gamma(C) * se + (ex * rel_e).sum(-1, keepdims=True)
        e_lse = e_se / se + 2 * U * np.abs(np.log(se)) + U * np.abs(lse)
        l_b = e_lse[:, 0] + U * np.abs(l)
        l = l * wv
        l_b = l_b * wv + U * np.abs(l)
        p = ex / se
        g = p - (np.arange(C)[None, :] == lab[:, None])
        e_g = p * (rel_e + e_se / se + 2 * U) + U * np.abs(g) + 2 * SUB
        acc = (z.argmax(-1).astype(np.float64) == t).astype(np.float64)
        acc_b = np.zeros(n)
        l = np.where(bad, np.nan, l)
        g = np.where(bad[:, None], np.nan, g)
        gi, e_gi = g, e_g
    else:
        t = f64(y).reshape(n, C)
        inv_out = 1.0 / C
        if kind == "bce_logits":
            L1 = np.log1p(np.exp(-np.abs(z)))
            term = np.maximum(z, 0) - z * t + L1
            e_term = U * np.abs(z * t) + 6 * U * L1 + U * (np.abs(np.maximum(z, 0) - z * t) + 2 * np.abs(term))
            sig = 1.0 / (1.0 + np.exp(-z))
            g = sig - t
            e_g = sig * 7 * U + U * np.abs(g) + np.where(sig < TINY, sig, 0.0)     # expf(-z) overflows: sigma = 0
        elif kind == "bce_probs":
            pc = np.clip(z, KERAS_EPS, ONE_M_EPS)
            la, lb = np.log(pc + KERAS_EPS), np.log(1.0 - pc + KERAS_EPS)
            term = -(t * la + (1.0 - t) * lb)
            e_la = 2 * U * np.abs(la) + U
            e_lb = 2 * U * np.abs(lb) + U + U * (1.0 - pc) / (1.0 - pc + KERAS_EPS)
            e_term = np.abs(t) * (e_la + U * np.abs(la)) + np.abs(1 - t) * (e_lb + U * np.abs(lb)) + 2 * U * np.abs(term)
            live = (z > KERAS_EPS) & (z < ONE_M_EPS)
            ga, gb = -t / (pc + KERAS_EPS), (1.0 - t) / (1.0 - pc + KERAS_EPS)
            g = np.where(live, ga + gb, 0.0)
            e_g = np.where(live, 4 * U * (np.abs(ga) + np.abs(gb)) + U * np.abs(g), 0.0)
        elif kind == "mse":
            d = z - t
            term = d * d
            e_term = 2 * np.abs(d) * U * np.abs(d) + U * term
            g = 2.0 * d
            e_g = 2 * U * np.abs(d)
        else:
            raise ValueError(kind)
        tw = term * wv[:, None]
        e_tw = (e_term + 4 * SUB) * wv[:, None] + U * np.abs(tw) + SUB
        l = tw.sum(-1) * inv_out
        l_b = (gamma(C) * np.abs(tw).sum(-1) + e_tw.sum(-1)) * inv_out + 2 * U * np.abs(l)
        hits = ((z > 0.5).astype(np.float64) == t).sum(-1)
        acc = hits * inv_out
        acc_b = np.zeros(n) if (C & (C - 1)) == 0 else 2 * U * np.abs(acc)
        gi = g * inv_out
        e_gi = e_g * inv_out + 2 * U * np.abs(gi)
    dz = gi * ib[:, None] * a
    dz_b = (np.abs(ib[:, None] * a) * (e_gi + SUB) + np.abs(gi * ib[:, None]) * e_a + np.abs(gi * a) * e_ib[:, None]
            + 2 * U * np.abs(dz) + 2 * SUB)
    lp, lpb = _block_sums(l, l_b, n)
    ap, apb = _block_sums(acc, acc_b, n)
    if not acc_b.any():
        apb = np.zeros_like(apb)
    return dict(row_loss=l, row_loss_bound=C_BOUND * l_b, row_acc=acc, row_acc_bound=C_BOUND * acc_b, dz=dz,
                dz_bound=C_BOUND * dz_b, loss_part=lp, loss_part_bound=C_BOUND * lpb, acc_part=ap, acc_part_bound=C_BOUND * apb)


# ---- positional encoding ----------------------------------------------------------------------------------------------
def pe(x, col_src, col_freq, col_begin, col_end, x_col_shift=0, row_index=None, col_feat=None, n_src=None, n=None):
    """dib_pe_kernel: out [n, col_end - col_begin] (column c - col_begin) and its bound.  row_index [nfeat, n] indexes x's rows
    per feature (clamped into [0, n_src))."""
    x = f64(x)
    n = x.shape[0] if n is None else n
    cols = np.arange(col_begin, col_end)
    out = np.zeros((n, len(cols)))
    bnd = np.zeros_like(out)
    for k, c in enumerate(cols):
        s = int(col_src[c])
        if s < 0:
            continue
        rows = np.arange(n)
        if row_index is not None:
            rows = np.clip(np.asarray(row_index)[int(col_feat[c])], 0, n_src - 1)
        xv = x[rows, s - x_col_shift]
        f = int(col_freq[c])
        if f == 0:
            out[:, k] = xv
        else:
            fx = f * xv
            out[:, k] = np.sin(fx)
            bnd[:, k] = np.abs(np.cos(fx)) * U * np.abs(fx) + 4 * U * np.abs(np.sin(fx)) + TINY
    return out, C_BOUND * bnd


# ---- dropout ----------------------------------------------------------------------------------------------------------
def dropout(x, keep, rate):
    """fl(x keep / (1 - rate)) on the kept columns, exactly as the kernel's one fp32 product (rate 0: x unchanged)"""
    x = np.asarray(x, np.float32)
    if rate <= 0:
        return x.astype(np.float64)
    inv_keep = np.float32(1.0) / (np.float32(1.0) - np.float32(rate))
    return np.where(keep, x * inv_keep, np.float32(0.0) * x).astype(np.float64)


# ---- stand-alone positional encoding ------------------------------------------------------------------------------------
def pe_plain(x, nfreq):
    """dib_pe_plain_kernel: x [n, d] -> [n, d nfreq] = [x | sin(2 x) | sin(4 x) | ...] and its bound"""
    x = f64(x)
    outs, bnds = [x], [np.zeros_like(x)]
    for k in range(1, nfreq):
        a = (2.0 ** k) * x
        outs.append(np.sin(a))
        bnds.append(C_BOUND * (4 * U * np.abs(np.sin(a)) + U * np.abs(np.cos(a)) * np.abs(a) + TINY))
    return np.concatenate(outs, -1), np.concatenate(bnds, -1)


# ---- optimizers -------------------------------------------------------------------------------------------------------
def adam(w, g, m, v, lr, t, b1, b2, eps):
    """one Keras-Adam update at step t (1-based) from fp32 w, g, m, v; returns (w', m', v') values and bounds"""
    w, g, m, v = f64(w), f64(g), f64(m), f64(v)
    b1, b2, eps, lr = (float(np.float32(a)) for a in (b1, b2, eps, lr))
    c1, c2 = 1.0 - b1, 1.0 - b2
    lr_t = lr * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    e_lr = 4 * U * lr_t
    m1 = m + (g - m) * c1
    e_m = 2 * U * np.abs(c1 * (g - m)) + U * np.abs(m1) + 2 * SUB
    v1 = v + (g * g - v) * c2
    e_v = c2 * (U * g * g + U * np.abs(g * g - v)) + U * np.abs(c2 * (g * g - v)) + U * np.abs(v1) + 3 * SUB
    sq = np.sqrt(v1)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_sq = np.minimum(np.where(sq > 0, e_v / (2 * sq), np.inf), np.sqrt(e_v)) + U * sq
    den = sq + eps
    q = lr_t * m1 / den
    e_q = (np.abs(m1) * e_lr + lr_t * e_m + U * np.abs(lr_t * m1) + np.abs(q) * (e_sq + U * den)) / den + U * np.abs(q)
    w1 = w - q
    return dict(w=w1, w_bound=C_BOUND * (e_q + U * np.abs(w1)), m=m1, m_bound=C_BOUND * e_m, v=v1, v_bound=C_BOUND * e_v)


def sgd(w, g, v, lr, momentum, nesterov):
    w, g, v = f64(w), f64(g), f64(v)
    lr, mo = float(np.float32(lr)), float(np.float32(momentum))
    lg = lr * g
    if mo == 0.0:
        w1 = w - lg
        return dict(w=w1, w_bound=C_BOUND * (U * np.abs(lg) + U * np.abs(w1)), v=v, v_bound=np.zeros_like(v))
    v1 = mo * v - lg
    e_v = U * (np.abs(mo * v) + np.abs(lg) + np.abs(v1))
    if nesterov:
        inner = mo * v1 - lg
        e_i = mo * e_v + U * (np.abs(mo * v1) + np.abs(lg) + np.abs(inner))
    else:
        inner, e_i = v1, e_v
    w1 = w + inner
    return dict(w=w1, w_bound=C_BOUND * (e_i + U * np.abs(w1)), v=v1, v_bound=C_BOUND * e_v)


def rmsprop(w, g, ms, mom, lr, rho, momentum, eps):
    w, g, ms, mom = f64(w), f64(g), f64(ms), f64(mom)
    lr, rho, mo, eps = (float(np.float32(a)) for a in (lr, rho, momentum, eps))
    c = 1.0 - rho
    ms1 = rho * ms + c * g * g
    e_ms = U * (np.abs(rho * ms) + 2 * c * g * g + np.abs(ms1))
    den = np.sqrt(ms1 + eps)
    e_den = (e_ms + U * (ms1 + eps)) / (2 * den) + U * den
    t = lr * g / den
    e_t = (U * np.abs(lr * g) + np.abs(t) * e_den) / den + U * np.abs(t)
    mom1 = mo * mom + t
    e_mo = U * np.abs(mo * mom) + e_t + U * np.abs(mom1)
    w1 = w - mom1
    return dict(w=w1, w_bound=C_BOUND * (e_mo + U * np.abs(w1)), ms=ms1, ms_bound=C_BOUND * e_ms, mom=mom1,
                mom_bound=C_BOUND * e_mo)


# ---- pairwise Gaussians -----------------------------------------------------------------------------------------------
def pairwise_gaussian(kind, ml1, ml2):
    """ml1 [n, 2E], ml2 [m, 2E] fp32 rows (mu | logvar) -> D [n, m] (kind 0 Bhattacharyya, 1 KL(1 || 2)), exp(-D), bounds"""
    ml1, ml2 = f64(ml1), f64(ml2)
    E = ml1.shape[1] // 2
    a, la = ml1[:, None, :E], ml1[:, None, E:]
    b, lb = ml2[None, :, :E], ml2[None, :, E:]
    d = a - b
    if kind == 0:
        sbar = 0.5 * (np.exp(la) + np.exp(lb))
        q = d * d / sbar
        x = 0.5 * np.abs(la - lb)
        lc = np.log1p(np.expm1(x) ** 2 / (2.0 * np.exp(x)))          # log cosh x, cosh x - 1 = expm1(x)^2 / (2 e^x)
        t1, t2 = q.sum(-1), lc.sum(-1)
        D = 0.125 * t1 + 0.5 * t2
        e_q = q * (8 * U + 5 * U) + U * q
        e_L = 5 * U + 2 * U * np.abs(np.log(sbar))
        e_t1 = gamma(E) * q.sum(-1) + e_q.sum(-1)
        e_t2 = gamma(3 * E) * (np.abs(np.log(sbar)) + 0.5 * np.abs(la) + 0.5 * np.abs(lb)).sum(-1) + e_L.sum(-1)
        e_D = 0.125 * e_t1 + 0.5 * e_t2 + U * np.abs(D)
    else:
        dl = la - lb
        ex = np.exp(dl)
        t2 = d * d * np.exp(-lb)
        D = 0.5 * (kl_r(dl) + t2).sum(-1)
        e_sub = (4 * U + U * np.abs(dl)) * ex + 8 * U * t2
        e_D = 0.5 * (gamma(5 * E) * (np.abs(lb) + np.abs(la) + 1.0 + ex + t2).sum(-1) + e_sub.sum(-1)) + U * np.abs(D)
    comp = np.exp(-D)
    e_c = comp * (np.expm1(C_BOUND * e_D) + 4 * U) + TINY
    return dict(D=D, D_bound=C_BOUND * e_D, comp=comp, comp_bound=C_BOUND * e_c)
