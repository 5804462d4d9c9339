"""TEST INFRASTRUCTURE ONLY -- a float64 reference of the InfoNCE kernels (csrc/dib_infonce_stream.cu, csrc/dib_infonce.cu)
with a worst-case error bound next to every output, derived from the fp32 arithmetic the kernels do.

From fp32 inputs e1 [n, d], e2 [n, d] and a temperature T it computes in float64
    s_ij = sim(e1_i, e2_j) / T,  r_i = log sum_j exp s_ij,  c_j = log sum_i exp s_ij,  s_ii,
    loss_sum = sum_i (r_i + c_i - 2 s_ii)  (= n * loss),
    d e1_i = sum_j w_ij d s_ij / d e1_i,  d e2_j = sum_i w_ij d s_ij / d e2_j,  w_ij = (p_ij + q_ij - 2 delta_ij) / n,
with p_ij = exp(s_ij - r_i), q_ij = exp(s_ij - c_j).  The similarities are the kernels' difference forms (l2 / l2sq sum
(a_k - b_k)^2; the reference's expanded |a|^2 + |b|^2 - 2ab is out of scope) with the kernels' fp32 epsilon.  'linf' follows
TF's reduce_max gradient: d s_ij is split evenly between the coordinates k attaining max_k |a_k - b_k|, ties decided on the
fp32-rounded |fl(a_k - b_k)| -- exactly the values the kernels compare.

Bounds (u = 2^-24, gamma_m = m u / (1 - m u); every bound below is the first-order sum of the rounding errors of the
kernels' operations, multiplied by C = C_BOUND = 2, which covers every product of two or more of them -- all first-order
terms here are < 1e-2, so the neglected terms are below 1 % of the bound):

sigma_ij, the error of one s_ij.  fl(a_k - b_k) is within u of the difference; the d-term fp32 accumulation in k order
(fmaf or add) of nonnegative terms is within gamma_d of their sum; sqrtf / division / the product with fl(1/T) each add u:
    l2sq  gamma_{d+4} D / T                         (D = sum_k (a_k - b_k)^2)
    l2    (gamma_{d+3} / 2 + gamma_3) |s|
    l1    gamma_{d+3} L1 / T
    linf  gamma_3 M / T                              (max is exact on the rounded |a_k - b_k|)
    cos   sigma_c / T + 2u |s|,  sigma_c = gamma_d sum_k |a_k b_k| / (|a| |b|) + (2 eps_n + 2u) |cos|,
          eps_n = gamma_d / 2 + u the relative error of a row norm (fmaf chain, then sqrtf).
    On operands on a grid of 2^-8 with |x| < 2^7 and T a power of two, float64 evaluates the kernels' l2sq / l1 / linf chains
    exactly; where every partial sum and the result are fp32 values, the kernel computes s_ij exactly: sigma_ij = 0 there.

rho_i, the error of one log-sum-exp.  log-sum-exp is 1-Lipschitz in the max norm, so the sigma's contribute max_j sigma_ij.
On the computed s the kernels add, per summed term: expf (2 ulp = 4u relative), the rounding of its argument (u |x| e^x <=
u relative to the running sum, which holds a term 1), one product and one add: 7u per term; a partial sum takes at most
`terms` = ceil(n / 32) terms (the streaming sweep: per lane; the head: per lane of a row, ceil(n / 8) per column group),
then a merge tree of <= 8 levels of the same form; logf adds 2u |log t| <= 2u log n, the final m + log t adds u |r|:
    rho_i = max_j sigma_ij + (7 terms + 56) u + 2u log n + u (|r_i| + max_j sigma_ij).

The error of one gradient element (i, k), with h_ijk = T d s_ij / d a_ik (a = the side's own rows, b = the other side):
    C [ gamma_m sum_j |w_ij h_ijk| + sum_j dw_ij |h_ijk| + sum_j |w_ij| E_ijk + 2u |sum_j w_ij h_ijk| ] / T
  * gamma_m: the fmaf accumulation over a tile of `tile` columns, then tile sums over ceil(n / tile) tiles
    (m = tile + ceil(n / tile); the streaming sweep tiles by 32, the head by 128);
  * dw_ij = [p_ij expm1(theta_p) + q_ij expm1(theta_q) + 2 tiny + 6u (p_ij + q_ij + 2 delta_ij)] / n, the error of one
    weight: theta_p = sigma_ij + rho_i + u (|s_ij - r_i| + sigma_ij + rho_i) + 4u (the perturbed exponent, its rounding,
    expf's 2 ulp), theta_q likewise with c_j; tiny = 2^-126 covers expf results below the normal range; 6u covers the add,
    the subtraction of 2, the product with fl(1/n) and, for linf, the product with fl(1 / ties);
  * E_ijk, the error of the kernels' per-pair factor: l2sq u |h|; l1 and linf 0 (the sign of fl(a - b) is exact);
    l2 (sigma_ij / |s_ij| + 4u) |h|; cosine [ |b_k| / |b| (2 eps_n + 5u) + |cos| |a_k| / |a| (2 eps_n + 10u)
    + sigma_c |a_k| / |a| ] / |a|;
  * 2u: the product with fl(1/T).
  The bound scales with sum_j |w h|, not with the max norm of the result, so the cancellation of sum_j w_ij ~ 0 is covered.

The loss sum: sum_i (rho_r_i + rho_c_i + 2 sigma_ii) + gamma_{ceil(rows / 256) + 16} sum_i (|r_i| + |c_i| + 2 |s_ii|).

Every function takes float32 arrays (the kernels' inputs) and returns float64.  The product path never imports this."""
from __future__ import annotations

import math

import numpy as np

from tests.fp_exact import C_BOUND, TINY, U, gamma, is_fp32


L2_EPS = float(np.float32(1e-9))           # kL2Eps of the kernels: utils.py's 1e-9 in fp32
KINDS = ("l2sq", "l2", "l1", "linf", "cosine")


def _on_exact_grid(x):
    x = np.asarray(x, dtype=np.float64)
    return bool(np.all(x * 256.0 == np.round(x * 256.0)) and np.all(np.abs(x) < 128.0))


def _is_pow2_float(t):
    return math.frexp(float(t))[0] == 0.5


class Pairs:
    """s_ij, sigma_ij and the per-pair derivative h_ijk = T d s_ij / d a_k with its error E_ijk, for fp32 rows a [m, d] against
    b [n, d].  The [m, n, d] tensors are formed for the rows given, so callers pass row blocks."""

    def __init__(self, a32, b32, kind, T, want_derivative=False):
        a32, b32 = np.asarray(a32, np.float32), np.asarray(b32, np.float32)
        a, b = a32.astype(np.float64), b32.astype(np.float64)
        d = a.shape[1]
        T = float(T)
        diff = a[:, None, :] - b[None, :, :]
        self.kind, self.T = kind, T
        if kind in ("l2sq", "l2"):
            D = (diff * diff).sum(-1)
            if kind == "l2sq":
                s, sig = -D / T, gamma(d + 4) * D / T
            else:
                R = np.sqrt(D + L2_EPS)
                s = -R / T
                sig = (gamma(d + 3) / 2 + gamma(3)) * np.abs(s)
        elif kind == "l1":
            L1 = np.abs(diff).sum(-1)
            s, sig = -L1 / T, gamma(d + 3) * L1 / T
        elif kind == "linf":
            M = np.abs(diff).max(-1)
            s, sig = -M / T, gamma(3) * M / T
        elif kind == "cosine":
            na, nb = np.linalg.norm(a, axis=-1), np.linalg.norm(b, axis=-1)
            cos = (a @ b.T) / (na[:, None] * nb[None, :])
            self.eps_n = gamma(d) / 2 + U
            self.sigma_c = gamma(d) * (np.abs(a) @ np.abs(b).T) / (na[:, None] * nb[None, :]) + (2 * self.eps_n + 2 * U) * np.abs(cos)
            s, sig = cos / T, self.sigma_c / T + 2 * U * np.abs(cos / T)
            self.cos, self.na, self.nb = cos, na, nb
        else:
            raise ValueError(kind)
        if kind in ("l2sq", "l1", "linf") and _is_pow2_float(T) and _on_exact_grid(a) and _on_exact_grid(b):
            # float64 evaluates the kernel's chain exactly here: where every partial value is an fp32 value, so is the kernel's
            if kind == "l2sq":
                part = np.cumsum(diff * diff, -1)
            elif kind == "l1":
                part = np.cumsum(np.abs(diff), -1)
            else:
                part = np.abs(diff)
            exact = is_fp32(part).all(-1) & is_fp32(diff).all(-1) & is_fp32(s) & ((s == 0) | (np.abs(s) >= 2.0 ** -126))
            sig = np.where(exact, 0.0, sig)
        self.s, self.sigma = s, sig
        if not want_derivative:
            return
        if kind == "l2sq":
            h = -2.0 * diff
            E = U * np.abs(h)
        elif kind == "l2":
            h = -diff / R[:, :, None]
            E = (sig / np.abs(s) + 4 * U)[:, :, None] * np.abs(h)
        elif kind == "l1":
            h = -np.sign(diff)
            E = np.zeros_like(h)
        elif kind == "linf":
            h = -np.sign(diff) * linf_tie_weights32(a32, b32)
            E = np.zeros_like(h)
        else:
            ah, bh = a / na[:, None], b / nb[:, None]
            h = (bh[None, :, :] - cos[:, :, None] * ah[:, None, :]) / na[:, None, None]
            en = self.eps_n
            E = (np.abs(bh)[None, :, :] * (2 * en + 5 * U) + (np.abs(cos)[:, :, None] * np.abs(ah)[:, None, :]) * (2 * en + 10 * U)
                 + self.sigma_c[:, :, None] * np.abs(ah)[:, None, :]) / na[:, None, None]
        self.h, self.E = h, E


def linf_tie_weights32(a32, b32):
    """[m, n, d]: 1 / (number of tied maxima) where |fl(a_k - b_k)| attains max_k, else 0 -- ties as the fp32 kernels see them."""
    ad = np.abs(np.asarray(a32, np.float32)[:, None, :] - np.asarray(b32, np.float32)[None, :, :])
    tied = ad == ad.max(-1, keepdims=True)
    return tied / tied.sum(-1, keepdims=True)


def _rho(s, sig, lse, n, terms, axis):
    ms = sig.max(axis)
    return ms + (7 * terms + 56) * U + 2 * U * math.log(max(n, 1)) + U * (np.abs(lse) + ms)


def lse_terms(n, head=False):
    """terms of the longest partial sum of one log-sum-exp: per lane of the streaming sweep, per column group of the head."""
    return -(-n // 8) if head else -(-n // 32)


def log_sum_exps(e1, e2, kind, T, head=False, chunk=256):
    """-> dict r, c, rho_r, rho_c, diag, sigma_diag over all n rows (row blocks of `chunk`; the [n, n] matrix never whole)."""
    n = e1.shape[0]
    r, rho_r = np.empty(n), np.empty(n)
    col_m, col_s, col_sig = np.full(n, -np.inf), np.zeros(n), np.zeros(n)
    diag, sdiag = np.empty(n), np.empty(n)
    terms = lse_terms(n, head)
    for i0 in range(0, n, chunk):
        P = Pairs(e1[i0:i0 + chunk], e2, kind, T)
        m = P.s.max(1)
        r[i0:i0 + chunk] = m + np.log(np.exp(P.s - m[:, None]).sum(1))
        rho_r[i0:i0 + chunk] = _rho(P.s, P.sigma, r[i0:i0 + chunk], n, terms, 1)
        cm = np.maximum(col_m, P.s.max(0))
        col_s = col_s * np.exp(col_m - cm) + np.exp(P.s - cm[None, :]).sum(0)
        col_m = cm
        col_sig = np.maximum(col_sig, P.sigma.max(0))
        idx = np.arange(i0, min(i0 + chunk, n))
        diag[idx], sdiag[idx] = P.s[idx - i0, idx], P.sigma[idx - i0, idx]
    c = col_m + np.log(col_s)
    rho_c = col_sig + (7 * terms + 56) * U + 2 * U * math.log(n) + U * (np.abs(c) + col_sig)
    return dict(r=r, c=c, rho_r=rho_r, rho_c=rho_c, diag=diag, sigma_diag=sdiag)


def loss_sum(lse, row0=0, rows=None):
    """(sum over the own rows of r_i + c_i - 2 s_ii, its bound)."""
    n = lse["r"].shape[0]
    rows = n - row0 if rows is None else rows
    sl = slice(row0, row0 + rows)
    r, c, dg = lse["r"][sl], lse["c"][sl], lse["diag"][sl]
    val = float((r + c - 2 * dg).sum())
    b = (lse["rho_r"][sl] + lse["rho_c"][sl] + 2 * lse["sigma_diag"][sl]).sum() + \
        gamma(-(-rows // 256) + 16) * (np.abs(r) + np.abs(c) + 2 * np.abs(dg)).sum()
    return val, C_BOUND * b


def _contract(w, h):
    """sum_j w_ij h_ijk as a batched matrix product"""
    return np.matmul(w[:, None, :], h)[:, 0, :]


def side_gradient(own, other, kind, T, lse_own, lse_other, rho_own, rho_other, row0=0, rows=None, tile=32, chunk=32,
                  parts=False):
    """d loss / d own_i for the own rows [row0, row0 + rows) against all n rows of `other` (own = e1 with lse_own = r,
    lse_other = c; own = e2 with lse_own = c, lse_other = r): -> (gradient [rows, d], bound [rows, d]).
    parts=True also returns the contribution of every 32-column tile [ceil(n / 32), rows, d] and of the diagonal's -2/n
    terms [rows, d]: the mutation check subtracts them (a kernel that left one out must leave the bounds)."""
    n, d = other.shape
    rows = n - row0 if rows is None else rows
    T = float(T)
    g, bnd = np.zeros((rows, d)), np.zeros((rows, d))
    nt = -(-n // 32)
    tiles = np.zeros((nt, rows, d)) if parts else None
    diag = np.zeros((rows, d)) if parts else None
    gm = gamma(tile + -(-n // tile))
    cols = np.arange(n)
    for i0 in range(row0, row0 + rows, chunk):
        i1 = min(i0 + chunk, row0 + rows)
        P = Pairs(own[i0:i1], other, kind, T, want_derivative=True)
        s, sig = P.s, P.sigma
        lo, lc = lse_own[i0:i1, None], lse_other[None, :]
        ro, rc = rho_own[i0:i1, None], rho_other[None, :]
        p, q = np.exp(s - lo), np.exp(s - lc)
        delta = (np.arange(i0, i1)[:, None] == cols[None, :]).astype(np.float64)
        w = (p + q - 2.0 * delta) / n
        tp = sig + ro + U * (np.abs(s - lo) + sig + ro) + 4 * U
        tq = sig + rc + U * (np.abs(s - lc) + sig + rc) + 4 * U
        dw = (p * np.expm1(tp) + q * np.expm1(tq) + 2 * TINY + 6 * U * (p + q + 2 * delta)) / n
        ah = np.abs(P.h)
        gc = _contract(w, P.h)
        b = gm * _contract(np.abs(w), ah) + _contract(dw, ah) + \
            _contract(np.abs(w), P.E) + 2 * U * np.abs(gc)
        g[i0 - row0:i1 - row0] = gc / T
        bnd[i0 - row0:i1 - row0] = C_BOUND * b / T
        if parts:
            for t in range(nt):
                tiles[t, i0 - row0:i1 - row0] = _contract(w[:, 32 * t:32 * t + 32], P.h[:, 32 * t:32 * t + 32]) / T
            diag[i0 - row0:i1 - row0] = _contract(-2.0 * delta / n, P.h) / T
    return (g, bnd, tiles, diag) if parts else (g, bnd)


def reference(e1, e2, kind, T, grads=True, head=False, **kw):
    """Everything at once for a full-range call: dict with the log_sum_exps entries, loss / loss_bound and, with grads,
    d1 / d1_bound / d2 / d2_bound."""
    lse = log_sum_exps(e1, e2, kind, T, head=head)
    out = dict(lse)
    out["loss"], out["loss_bound"] = loss_sum(lse)
    if grads:
        tile = 128 if head else 32
        out["d1"], out["d1_bound"] = side_gradient(e1, e2, kind, T, lse["r"], lse["c"], lse["rho_r"], lse["rho_c"], tile=tile, **kw)
        out["d2"], out["d2_bound"] = side_gradient(e2, e1, kind, T, lse["c"], lse["r"], lse["rho_c"], lse["rho_r"], tile=tile, **kw)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the cases the kernel tests run (tests/test_gpu_infonce_stream.py); the mutation check of the host test runs the same
# ---------------------------------------------------------------------------------------------------------------------
# (n, d) of the gradient checks: every d of {1, 2, 3, 31, 32, 33, 64, 127, 128, 255, 257, 511, 512} at an n that is not a
# multiple of 32, and every n of {1, 2, 31, 32, 33, 63, 65, 100, 1000, 4097} with widths on both sides of 32 (4097 only
# with narrow ones: the float64 reference forms [rows, n, d] pair tensors on the CPU)
GRAD_SHAPES = [(1, 3), (1, 64), (2, 1), (2, 33), (31, 31), (31, 2), (32, 33), (32, 3), (33, 32), (33, 1), (63, 127), (63, 31),
               (65, 128), (65, 33), (100, 255), (100, 32), (65, 257), (33, 511), (100, 512), (1000, 64), (1000, 31),
               (1000, 33), (4097, 3), (4097, 2)]
REGIMES = ("normal", "wide", "peaked", "identical", "duplicate", "dyadic")


def case_data(kind, n, d, regime="normal", T=1.0, seed=0):
    """fp32 e1, e2 [n, d] and the temperature of one case.
    normal     e2 = e1 + noise, logits spanning about 4
    wide       logits spanning well over 200 at the given T (cosine at T = 2^-8: |s| <= 1/T), so exp underflows in a row
    peaked     e2 = e1 on well separated rows: each softmax sits on its diagonal and w_ii ~ 0 by cancellation
    identical  every row of e1 the same, every row of e2 the same
    duplicate  e2_j = e1_{j+1} for even j: pairs i != j at distance 0 (the l2 epsilon, sign(0) for l1 / linf)
    dyadic     multiples of 1/4 in [-2, 2], T a power of two: exact l2sq / l1 / linf similarities, linf ties everywhere"""
    rng = np.random.default_rng([seed, n, d, KINDS.index(kind), REGIMES.index(regime)])
    x = rng.standard_normal((n, d))
    if kind == "cosine" and regime in ("wide", "peaked"):
        T = 2.0 ** -8
    if regime == "dyadic":
        e1 = rng.integers(-8, 9, size=(n, d)) / 4.0
        e2 = rng.integers(-8, 9, size=(n, d)) / 4.0
        e2[::3] = e1[::3]
        return e1.astype(np.float32), e2.astype(np.float32), T
    if regime == "identical":
        return (np.repeat(x[:1], n, 0).astype(np.float32), np.repeat(rng.standard_normal((1, d)), n, 0).astype(np.float32), T)
    e1 = x / math.sqrt(d)
    e2 = e1 + 0.5 * rng.standard_normal((n, d)) / math.sqrt(d)
    if regime == "duplicate":
        e2[0:n - 1:2] = e1[1:n:2]
    if regime == "peaked":
        e2 = e1 + 1e-3 * rng.standard_normal((n, d)) / math.sqrt(d)
    if kind != "cosine" and n > 1:
        S = Pairs(e1.astype(np.float32)[:64], e2.astype(np.float32), kind, T).s
        span = S.max() - S.min()
        if span > 0:
            f = (300.0 if regime in ("wide", "peaked") else 4.0) / span
            f = math.sqrt(f) if kind == "l2sq" else f
            e1, e2 = e1 * f, e2 * f
    return e1.astype(np.float32), e2.astype(np.float32), T
