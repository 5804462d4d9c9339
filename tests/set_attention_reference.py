"""TEST INFRASTRUCTURE ONLY -- a float64 reference of the set-transformer kernels (csrc/dib_set_attn.cu: fixed-size attention,
LayerNorm, mean pooling; csrc/dib_set_attn_varlen.cu: key-tiled masked attention, masked pooling, zero_pad_rows) with a
worst-case error bound next to every output, derived from the fp32 arithmetic the kernels do.

Attention works on one (set, head) at a time in the head-split layout [sets, heads, L, dk]; set s has l_s real rows (the
fixed-size kernels: l_s = L), keys j >= l_s are masked out and padding query rows are exactly 0 in every output.

Inputs are restated exactly where numpy float32 can: the kernels scale q by the fp32 value c = fl(1 / sqrtf(dk)) into
q~ = fl(q c) (load_rows / load_tile), and the reference starts from that same fp32 q~.  fp32 inputs are the kernels'; float64
inputs (the model oracles') are scaled by the exact 1 / sqrt(dk) instead.  Everything after that is float64:
    s_ij = sum_d q~_id k_jd,  P_ij = softmax_j s_ij,  lse_i = log sum_j exp s_ij,  O = P V.
The backward, like the kernels, recomputes P from the lse it is GIVEN (lambda, an fp32 array) and reads the given o:
    P'_ij = exp(s_ij - lambda_i),  D_i = sum_d dO_id o_id,  dP = dO V^T,  dS = P' o (dP - D),
    dV = P'^T dO,  dQ = c dS K,  dK = dS^T Q~.

Bounds.  u = 2^-24, gamma_m = m u / (1 - m u).  Each bound is C = C_BOUND = 2 times the first-order sum of the rounding errors
of the kernel's own fp32 operations (the factor 2 covers every product of two or more of them; every first-order term here
is far below 1e-2).  expf has an error of 2 ulp (4u relative), logf 1 ulp; the library is built without fast-math.  Every
sum is bounded by gamma_m sum |terms| plus the propagated errors of its terms, never by the size of its result, so sums that
cancel (dS: sum_j P_ij (dP_ij - D_i) = 0; the LayerNorm backward) are covered.  Each term below names the kernel function
and the statement it follows (dib_set_attn.cu: the fixed-size kernels; dib_set_attn_varlen.cu: varlen).

  sigma_ij, one score (fixed scores(); varlen tile_dots(): an fmaf chain in d order):  gamma_dk sum_d |q~_id k_jd|.  Zero
    where every partial sum of the chain is an fp32 value (dyadic operands; dk in {1, 4, 16, 64} makes c a power of two).
  The softmax of row i (span_i = max_j s_ij - min_j s_ij over the real keys, sigma^_i = max_j sigma_ij):
    fixed (attn_fwd_kernel): e_j = expf(fl(s_j - m)) -- u (span + 2 sigma^) for the argument, 4u for expf; a lane sum of
      ceil(L / 32) terms and a 5-level shuffle tree: gamma_{ceil(L/32) + 5}; then fl(1 / sum) and fl(e inv): 2u.
      eps_w = u (span + 2 sigma^) + 4u,  gamma_sum = gamma_{ceil(L/32) + 5},  O: an fmaf chain of L terms, gamma_L.
    varlen (attn_varlen_fwd_kernel): per 64-key tile (nT = ceil(l / 64) tiles) p = expf(s - mn), the running maximum's
      alpha = expf(m - mn), o *= alpha and lsum = fmaf(lsum, alpha, tile sum): every term meets at most nT exponentials and
      nT rescales, eps_w = nT (u (span + 2 sigma^) + 5u); a tile sum is 3 adds and a 4-level half-warp tree and the tiles
      merge by fmaf: gamma_sum = gamma_{8 + nT}; O: fmaf chains over the l keys plus nT rescales, gamma_{l + nT}; then
      fl(1 / lsum) and fl(o inv): 2u.
    The relative error of one weight P_ij is then eps_p = expm1(sigma_ij + sigma^_i) + eps_w + (eps_w + gamma_sum) + 2u
    (score errors move log P by at most sigma_ij + sigma^_i: lse is 1-Lipschitz in the max norm); an exponential that
    underflows adds 2 tiny (tiny = 2^-126) absolutely.
      O_id:   gamma_acc sum_j P_ij |v_jd| + sum_j (P_ij eps_p_ij + 2 tiny) |v_jd|
      lse_i:  sigma^_i + eps_w + gamma_sum + 2u log l + u (|lse_i| + sigma^_i) + tiny   (lse = fl(m + logf(sum)))
    At l = 1 both kernels compute p = 1 exactly: O = V and lse = s_00 (bound sigma_00).
  The backward (attn_bwd_kernel; varlen attn_varlen_bwd_dq_kernel / attn_varlen_bwd_dkdv_kernel):
      P'_ij:  expf(fl(s~_ij - lambda_i)): P' (expm1(sigma_ij + u (|s_ij - lambda_i| + sigma_ij)) + 4u) + tiny
      D_i:    lane-strided fmaf chains of ceil(dk / 32) terms and a 5-level tree: gamma_{ceil(dk/32) + 5} sum_d |dO_id o_id|
      dP_ij:  gamma_dk sum_d |dO_id v_jd|
      dS_ij = fl(p fl(dP - D)):  P' (e_dP + e_D + u |dP - D|) + e_P' |dP - D| + u |dS|
      dV_jd:  gamma_l sum_i P'_ij |dO_id| + sum_i e_P'_ij |dO_id|              (fixed: gamma_L, a chain over all L rows)
      dQ_id:  c (gamma_l sum_j |dS_ij k_jd| + sum_j e_dS_ij |k_jd|) + u |dQ_id|  (the chain, then fl(. c))
      dK_jd:  gamma_l sum_i |dS_ij q~_id| + sum_i e_dS_ij |q~_id|
      dsum_i (varlen): the D_i above.

LayerNorm (ln_fwd_kernel / ln_bwd_kernel; one warp per row, 4 columns per lane), z = a + b in float64:
  forward: z~ = fl(a + b): u |z|; the mean: a lane sum of 4 and a 5-level tree, then / E:
      e_mu = (gamma_8 + u) sum_e |z_e| / E + u |mu|;  e_c_e = u |z_e| + e_mu + u |c_e|  (c = z - mu, fl(z~ - mu~));
      the variance: fmaf chains of 4 and a 5-level tree, / E, + eps: e_w = (gamma_9 sum c^2 + sum (2 |c| e_c + e_c^2)) / E
      + 2u (var + eps)  -- the square e_c^2 is kept: for a constant row (var = 0) it is all there is;
      rstd = fl(1 / sqrtf(w)): e_r = r (e_w / (2 w) + 2u);
      y = fl(fl(fl(c~ r~) gamma) + beta): |gamma| (r e_c + |c| e_r + u |xh|) + u |xh gamma| + u |y|.
  backward, from the GIVEN mean m and rstd r: xh = (z - m) r, e_xh = r (u |z| + u |z - m|) + u |xh|;
      dy = the pooled term fl(dy_pool fl(1 / pool_rows)) (or fl(1 / l_s) on the real rows) plus up to 4 sources:
      e_dy = gamma_5 sum |terms|;  g = fl(dy gamma): e_g = |gamma| e_dy + u |g|;
      m1 = mean(g), m2 = mean(g xh): lane chains of 4 and a 5-level tree, / E:
      e_m1 = (gamma_9 sum |g| + sum e_g) / E + u |m1|,  e_m2 = (gamma_9 sum |g xh| + sum (e_g |xh| + |g| e_xh)) / E + u |m2|;
      dz = fl(r fl(fl(g - m1) - fl(xh m2))): r (e_g + e_m1 + u |g - m1| + e_xh |m2| + |xh| e_m2 + u |xh m2| + u |inner|)
      + u |dz|;  d_branch = fl(dz act'(b)) with act' from the output b (dib_act_grad): |act'| e_dz + |dz| e_act + u |dz act'|,
      e_act = u |b^2| + u |1 - b^2| (tanh), 2u |b (1 - b)| (sigmoid), u |b + 1| (elu, b <= 0), else 0;
      d gamma / d beta partials of split s: per warp an fmaf chain over ceil(n_s / 8) rows, then the 8 warps' sum in warp
      order: gamma_{ceil(n_s/8) + 8} sum |dy xh| + sum (e_dy |xh| + |dy| e_xh)  (d beta: with xh = 1, e_xh = 0).

Pooling (pool_fwd_kernel / pool_varlen_fwd_kernel): acc += x over the l rows, then acc / l:
      gamma_l sum_p |x_p| / l + u |out|;  exactly 0 where every partial sum is an fp32 value and l is a power of two.

round_out is cvt.rna.tf32.f32 applied to an output: round_tf32 (the grouped-GEMM tests' restatement, imported, not copied).
Every function returns float64 arrays.  The product path never imports this."""
from __future__ import annotations

import math

import numpy as np

from tests.test_gpu_grouped_gemm import round_tf32  # noqa: F401  (re-exported: the rna rounding of round_out)

U = 2.0 ** -24
C_BOUND = 2.0
TINY = 2.0 ** -126
ACTS = ("linear", "relu", "tanh", "leaky_relu", "sigmoid", "elu")


def gamma(m):
    m = np.asarray(m, np.float64)
    return m * U / (1.0 - m * U)


def scale32(dk):
    """fl(1 / sqrtf(dk)), the kernels' fp32 scale"""
    return np.float32(1.0) / np.sqrt(np.float32(dk))


def _is_fp32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64) == x


def _on_grid(x):
    """multiples of 2^-12 below 2^8: products and sums of up to 128 of them are exact in float64"""
    x = np.asarray(x, np.float64)
    return bool(np.all(x * 4096.0 == np.round(x * 4096.0)) and np.all(np.abs(x) < 256.0))


def _pow2(n):
    return (np.asarray(n) & (np.asarray(n) - 1)) == 0


def split_heads(x, sets, L, heads, dk):
    """[sets * L, >= heads * dk] rows -> [sets, heads, L, dk]"""
    x = np.asarray(x)[:, :heads * dk]
    return x.reshape(sets, L, heads, dk).transpose(0, 2, 1, 3)


def merge_heads(x):
    """[sets, heads, L, dk] -> [sets * L, heads * dk]"""
    S, H, L, dk = x.shape
    return x.transpose(0, 2, 1, 3).reshape(S * L, H * dk)


def _scaled_q(q, dk):
    q = np.asarray(q)
    if q.dtype == np.float32:
        return (q * scale32(dk)).astype(np.float64)
    return q.astype(np.float64) / math.sqrt(dk)


def _sizes(sizes, S, L):
    """per-set real rows [S] (None: the fixed-size kernels, l = L) and the masks [S, 1, L, 1] (rows) / [S, 1, 1, L] (keys)"""
    l = np.full(S, L, np.int64) if sizes is None else np.clip(np.asarray(sizes, np.int64), 1, L)
    real = np.arange(L)[None, :] < l[:, None]
    return l, real[:, None, :, None], real[:, None, None, :]


def scores(qs, k, sizes=None):
    """s [S, H, L, L] (masked keys -inf) and sigma (0 where the fmaf chain in d order is exact)"""
    S, H, L, dk = qs.shape
    k = np.asarray(k, np.float64)
    s = qs @ k.swapaxes(-1, -2)
    sig = gamma(dk) * (np.abs(qs) @ np.abs(k).swapaxes(-1, -2))
    if _on_grid(qs) and _on_grid(k) and S * H * L * L * dk <= 2 ** 24:
        # float64 forms every partial sum of the chain exactly here; where each is an fp32 value, so is the kernel's
        part = np.zeros_like(s)
        exact = np.ones(s.shape, bool)
        for d in range(dk):
            part = part + qs[..., :, None, d] * k[..., None, :, d]
            exact &= _is_fp32(part)
        sig = np.where(exact, 0.0, sig)
    _, _, kreal = _sizes(sizes, S, L)
    return np.where(kreal, s, -np.inf), np.where(kreal, sig, 0.0)


def attention_forward(q, k, v, sizes=None):
    """q, k, v [S, H, L, dk] (fp32: the kernels' inputs; float64: exact scaling); sizes None = the fixed-size kernel.
    -> dict o, o_bound [S, H, L, dk], lse, lse_bound [S, H, L] (bounds already times C_BOUND), s, sigma."""
    S, H, L, dk = np.shape(q)
    l, rreal, kreal = _sizes(sizes, S, L)
    q, k, v = (np.where(rreal, t, np.zeros((), np.asarray(t).dtype)) for t in (q, k, v))   # padding rows are never read
    qs = _scaled_q(q, dk)
    v = np.asarray(v, np.float64)
    s, sig = scores(qs, k, sizes)
    m = s.max(-1, keepdims=True)
    e = np.exp(s - m)
    ssum = e.sum(-1, keepdims=True)
    P = e / ssum
    lse = (m + np.log(ssum))[..., 0]
    o = P @ v
    sfin = np.where(kreal, s, np.nan)
    span = (np.nanmax(sfin, -1) - np.nanmin(sfin, -1))[..., None]
    sh = sig.max(-1, keepdims=True)
    lb = l[:, None, None, None].astype(np.float64)
    if sizes is None:
        eps_w = U * (span + 2 * sh) + 4 * U
        g_sum, g_acc = gamma(-(-L // 32) + 5), gamma(L)
    else:
        nT = np.ceil(lb / 64)
        eps_w = nT * (U * (span + 2 * sh) + 5 * U)
        g_sum, g_acc = gamma(8 + nT), gamma(lb + nT)
    eps_p = np.expm1(sig + sh) + 2 * eps_w + g_sum + 2 * U
    dp = np.where(kreal, P * eps_p + 2 * TINY, 0.0)
    va = np.abs(v)
    ob = g_acc * (P @ va) + dp @ va
    lb_ = (sh + eps_w + g_sum + 2 * U * np.log(lb) + U * (np.abs(lse[..., None]) + sh) + TINY)[..., 0]
    one = (l == 1)[:, None, None]
    ob = np.where(one[..., None], 0.0, ob)
    lb_ = np.where(one, sig[..., 0], lb_)
    o = np.where(rreal, o, 0.0)
    lse = np.where(rreal[..., 0], lse, 0.0)
    return dict(o=o, o_bound=C_BOUND * np.where(rreal, ob, 0.0), lse=lse, lse_bound=C_BOUND * np.where(rreal[..., 0], lb_, 0.0),
                s=s, sigma=sig, P=np.where(rreal, P, 0.0))


def attention_backward(q, k, v, dout, o, lse, sizes=None, mutate=None):
    """From the GIVEN o [S, H, L, dk] and lse [S, H, L] (what the kernels read): -> dict dq, dk, dv, dsum and their bounds.
    mutate (host mutation checks only): 'no_D' drops -D from dS, 'no_scale' drops the 1/sqrt(dk) of dQ."""
    S, H, L, dk = np.shape(q)
    l, rreal, kreal = _sizes(sizes, S, L)
    q, k, v, dout, o = (np.where(rreal, t, np.zeros((), np.asarray(t).dtype)) for t in (q, k, v, dout, o))
    qs = _scaled_q(q, dk)
    c = float(scale32(dk)) if np.asarray(q).dtype == np.float32 else 1.0 / math.sqrt(dk)
    k, v = np.asarray(k, np.float64), np.asarray(v, np.float64)
    g, o = np.asarray(dout, np.float64), np.asarray(o, np.float64)
    lam = np.where(rreal[..., 0], np.asarray(lse, np.float64), 0.0)[..., None]
    s, sig = scores(qs, k, sizes)
    both = rreal & kreal
    arg = np.where(both, s - lam, -np.inf)
    Pp = np.exp(arg)
    eP = np.where(both, Pp * (np.expm1(sig + U * (np.abs(np.where(both, arg, 0.0)) + sig)) + 4 * U) + TINY, 0.0)
    D = (g * o).sum(-1, keepdims=True)
    eD = gamma(-(-dk // 32) + 5) * (np.abs(g) * np.abs(o)).sum(-1, keepdims=True)
    dP = g @ v.swapaxes(-1, -2)
    edP = gamma(dk) * (np.abs(g) @ np.abs(v).swapaxes(-1, -2))
    diff = dP - (0.0 if mutate == "no_D" else D)
    dS = np.where(both, Pp * diff, 0.0)
    edS = np.where(both, Pp * (edP + eD + U * np.abs(dP - D)) + eP * np.abs(dP - D) + U * np.abs(dS), 0.0)
    lb = l[:, None, None, None].astype(np.float64)
    g_acc = gamma(L) if sizes is None else gamma(lb)
    ga, ka, qa = np.abs(g), np.abs(k), np.abs(qs)
    dv = Pp.swapaxes(-1, -2) @ g
    dv_b = g_acc * (Pp.swapaxes(-1, -2) @ ga) + eP.swapaxes(-1, -2) @ ga
    cq = 1.0 if mutate == "no_scale" else c
    dq = cq * (dS @ k)
    dq_b = c * (g_acc * (np.abs(dS) @ ka) + edS @ ka) + U * np.abs(dq)
    dkk = dS.swapaxes(-1, -2) @ qs
    dk_b = g_acc * (np.abs(dS).swapaxes(-1, -2) @ qa) + edS.swapaxes(-1, -2) @ qa
    z = lambda t: np.where(rreal, t, 0.0)
    return dict(dq=z(dq), dq_bound=C_BOUND * z(dq_b), dk=z(dkk), dk_bound=C_BOUND * z(dk_b), dv=z(dv), dv_bound=C_BOUND * z(dv_b),
                dsum=np.where(rreal[..., 0], D[..., 0], 0.0), dsum_bound=C_BOUND * np.where(rreal[..., 0], eD[..., 0], 0.0),
                dS=dS, P=Pp)


def layer_norm_forward(a, b, gamma_, beta, eps):
    """a, b [rows, E]; -> dict y, mean, rstd and their bounds"""
    z = np.asarray(a, np.float64) + np.asarray(b, np.float64)
    E = z.shape[1]
    ga, be = np.asarray(gamma_, np.float64), np.asarray(beta, np.float64)
    eps = float(np.float32(eps))
    mu = z.mean(1, keepdims=True)
    c = z - mu
    var = (c * c).mean(1, keepdims=True)
    w = var + eps
    r = 1.0 / np.sqrt(w)
    xh = c * r
    y = xh * ga + be
    e_mu = (gamma(8) + U) * np.abs(z).sum(1, keepdims=True) / E + U * np.abs(mu)
    e_c = U * np.abs(z) + e_mu + U * np.abs(c)
    e_w = (gamma(9) * (c * c).sum(1, keepdims=True) + (2 * np.abs(c) * e_c + e_c * e_c).sum(1, keepdims=True)) / E + 2 * U * w
    e_r = r * (e_w / (2 * w) + 2 * U)
    e_y = np.abs(ga) * (r * e_c + np.abs(c) * e_r + U * np.abs(xh)) + U * np.abs(xh * ga) + U * np.abs(y)
    return dict(y=y, y_bound=C_BOUND * e_y, mean=mu[:, 0], mean_bound=C_BOUND * e_mu[:, 0], rstd=r[:, 0],
                rstd_bound=C_BOUND * e_r[:, 0])


def act_grad(act, h, alpha):
    """dib_act_grad in float64 from the output h, and the error of its fp32 evaluation"""
    h = np.asarray(h, np.float64)
    if act == "relu":
        return (h > 0).astype(np.float64), np.zeros_like(h)
    if act == "tanh":
        return 1.0 - h * h, U * h * h + U * np.abs(1.0 - h * h)
    if act == "leaky_relu":
        return np.where(h > 0, 1.0, float(np.float32(alpha))), np.zeros_like(h)
    if act == "sigmoid":
        return h * (1.0 - h), 2 * U * np.abs(h * (1.0 - h))
    if act == "elu":
        return np.where(h > 0, 1.0, h + 1.0), np.where(h > 0, 0.0, U * np.abs(h + 1.0))
    return np.ones_like(h), np.zeros_like(h)


def pooled_dy(dy_pool, rows, pool_rows, sizes=None, divide_by_lmax=False):
    """the pooled source of every row [rows, E]: dy_pool[r / pool_rows] fl(1 / pool_rows), or fl(1 / l_s) on the real rows
    (divide_by_lmax: the host mutation check's wrong divisor)"""
    dp = np.asarray(dy_pool, np.float64)
    s = np.arange(rows) // pool_rows
    if sizes is None or divide_by_lmax:
        real = np.ones(rows, bool) if sizes is None else (np.arange(rows) % pool_rows) < np.clip(np.asarray(sizes), 1, pool_rows)[s]
        return np.where(real[:, None], dp[s] * float(np.float32(1) / np.float32(pool_rows)), 0.0)
    l = np.clip(np.asarray(sizes, np.int64), 1, pool_rows)[s]
    real = (np.arange(rows) % pool_rows) < l
    inv = (np.float32(1) / l.astype(np.float32)).astype(np.float64)
    return np.where(real[:, None], dp[s] * inv[:, None], 0.0)


def layer_norm_backward(a, b, gamma_, mean, rstd, dys=(), pooled=None, branch_act=None, alpha=0.2, nsplit=1, rows_per_split=None):
    """From the GIVEN mean / rstd [rows]: dys = the per-row sources [rows, E], pooled = pooled_dy(...) or None ->
    dict d_res, d_branch (None without branch_act), dgamma / dbeta partials [nsplit, E], and their bounds."""
    z = np.asarray(a, np.float64) + np.asarray(b, np.float64)
    rows, E = z.shape
    ga = np.asarray(gamma_, np.float64)
    m, r = np.asarray(mean, np.float64)[:, None], np.asarray(rstd, np.float64)[:, None]
    xh = (z - m) * r
    e_xh = r * (U * np.abs(z) + U * np.abs(z - m)) + U * np.abs(xh)
    terms = [np.asarray(t, np.float64) for t in dys] + ([pooled] if pooled is not None else [])
    dy = sum(terms) if terms else np.zeros_like(z)
    e_dy = gamma(5) * sum(np.abs(t) for t in terms) if terms else np.zeros_like(z)
    gg = dy * ga
    e_g = np.abs(ga) * e_dy + U * np.abs(gg)
    m1 = gg.mean(1, keepdims=True)
    m2 = (gg * xh).mean(1, keepdims=True)
    e_m1 = (gamma(9) * np.abs(gg).sum(1, keepdims=True) + e_g.sum(1, keepdims=True)) / E + U * np.abs(m1)
    e_m2 = (gamma(9) * np.abs(gg * xh).sum(1, keepdims=True) + (e_g * np.abs(xh) + np.abs(gg) * e_xh).sum(1, keepdims=True)) / E \
        + U * np.abs(m2)
    inner = gg - m1 - xh * m2
    dz = r * inner
    e_dz = r * (e_g + e_m1 + U * np.abs(gg - m1) + e_xh * np.abs(m2) + np.abs(xh) * e_m2 + U * np.abs(xh * m2) + U * np.abs(inner)) \
        + U * np.abs(dz)
    out = dict(d_res=dz, d_res_bound=C_BOUND * e_dz, d_branch=None, d_branch_bound=None)
    if branch_act is not None:
        ag, e_ag = act_grad(branch_act, b, alpha)
        out["d_branch"] = dz * ag
        out["d_branch_bound"] = C_BOUND * (np.abs(ag) * e_dz + np.abs(dz) * e_ag + U * np.abs(dz * ag))
    rps = rows if rows_per_split is None else rows_per_split
    dg, db = np.zeros((nsplit, E)), np.zeros((nsplit, E))
    dgb, dbb = np.zeros((nsplit, E)), np.zeros((nsplit, E))
    for s in range(nsplit):
        r0, r1 = min(s * rps, rows), min((s + 1) * rps, rows)
        if r1 <= r0:
            continue
        gm = gamma(-(-(r1 - r0) // 8) + 8)
        sl = slice(r0, r1)
        dg[s] = (dy[sl] * xh[sl]).sum(0)
        db[s] = dy[sl].sum(0)
        dgb[s] = gm * np.abs(dy[sl] * xh[sl]).sum(0) + (e_dy[sl] * np.abs(xh[sl]) + np.abs(dy[sl]) * e_xh[sl]).sum(0)
        dbb[s] = gm * np.abs(dy[sl]).sum(0) + e_dy[sl].sum(0)
    out.update(dgamma=dg, dgamma_bound=C_BOUND * dgb, dbeta=db, dbeta_bound=C_BOUND * dbb)
    return out


def pool(x, L, sizes=None):
    """x [sets * L, E] -> (the mean over each set's l_s real rows [sets, E], its bound; 0 where the kernel is exact)"""
    x = np.asarray(x, np.float64)
    S, E = x.shape[0] // L, x.shape[1]
    xs = x.reshape(S, L, E)
    l = np.full(S, L, np.int64) if sizes is None else np.clip(np.asarray(sizes, np.int64), 1, L)
    real = (np.arange(L)[None, :] < l[:, None])[..., None]
    xr = np.where(real, xs, 0.0)
    out = xr.sum(1) / l[:, None]
    part = np.cumsum(xr, 1)
    exact = _is_fp32(part).all(1) & _pow2(l)[:, None] & ((out == 0) | (np.abs(out) >= 2.0 ** -126))
    b = gamma(l)[:, None] * np.abs(xr).sum(1) / l[:, None] + U * np.abs(out)
    return out, C_BOUND * np.where(exact, 0.0, b)


# ---------------------------------------------------------------------------------------------------------------------
# the cases the kernel tests run (tests/test_gpu_set_attention_kernels.py); the host test's mutation checks run the same
# ---------------------------------------------------------------------------------------------------------------------
REGIMES = ("normal", "wide", "peaked", "flat", "identical", "dyadic")


def attention_case(S, H, L, dk, regime="normal", seed=0):
    """fp32 q, k, v, dout [S, H, L, dk] of one case.
    normal     logits spanning about 8 in a row
    wide       logits spanning well over 100 in a row (exp underflows)
    peaked     q_i a large multiple of k_i: each softmax sits on its own key
    flat       q = 0: every score is exactly 0
    identical  every key of a (set, head) the same
    dyadic     multiples of 1/4 in [-2, 2]: exact scores (sigma = 0) for dk in {1, 4, 16, 64}"""
    rng = np.random.default_rng([seed, S, H, L, dk, REGIMES.index(regime)])
    shape = (S, H, L, dk)
    if regime == "dyadic":
        q, k, v, g = (rng.integers(-8, 9, size=shape) / 4.0 for _ in range(4))
        return tuple(t.astype(np.float32) for t in (q, k, v, g))
    q, k, v, g = (rng.standard_normal(shape) for _ in range(4))
    f = {"normal": 2.0, "wide": 40.0, "peaked": 6.0}.get(regime, 1.0)
    if regime == "peaked":
        q = f * k * math.sqrt(dk) / np.maximum(np.linalg.norm(k, axis=-1, keepdims=True), 1e-3) + 0.1 * q
    elif regime == "flat":
        q = np.zeros(shape)
    elif regime == "identical":
        k = np.repeat(k[:, :, :1], L, 2)
        q = 2.0 * q
    else:
        q = f * q
    return tuple(t.astype(np.float32) for t in (q, k, v, g))
