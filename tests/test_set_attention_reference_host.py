"""CPU checks of the float64 set-transformer kernel reference (tests/set_attention_reference.py): it agrees with the model
oracles and with torch autograd, its bounds vanish only where the kernels' arithmetic is exact, and they are tight enough that
a kernel with one of the seeded faults below would leave them."""
import math

import numpy as np
import pytest
import torch

from tests import set_attention_reference as R
from tests import set_transformer_oracle as STO
from tests import set_transformer_varlen_oracle as VO

SMALL = STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[8], bottleneck_dimension=8, number_particles=6,
                     key_dim=4, number_heads=2, number_attention_blocks=1, ff_arch_per_block=[16, 8], final_processing_arch=[6],
                     number_positional_encoding_frequencies=3)


def _model_case(sizes):
    rng = np.random.default_rng(3)
    B, L = len(sizes), SMALL.number_particles
    p = STO.init_params(SMALL, rng, dtype=np.float64)
    x = rng.standard_normal((B, L, SMALL.particle_feature_dimensions))
    eps = rng.standard_normal((B, L, SMALL.bottleneck_dimension))
    return p, x, eps


@pytest.mark.parametrize("sizes", [None, [1, 6, 3, 5]])
def test_attention_and_layer_norm_agree_with_the_model_oracles(sizes):
    p, x, eps = _model_case([6] * 4 if sizes is None else sizes)
    fr = STO.forward(SMALL, p, x, eps, keep=True) if sizes is None else VO.forward(SMALL, p, x, eps, sizes, keep=True)
    bc = fr.cache["bc"][0]
    dk = SMALL.key_dim
    ref = R.attention_forward(bc["Q"] * math.sqrt(dk), bc["K"], bc["V"], sizes)
    np.testing.assert_allclose(ref["o"], STO._heads(bc["O"], SMALL.number_heads, dk), rtol=0, atol=1e-12)
    np.testing.assert_allclose(ref["P"], bc["P"], rtol=0, atol=1e-12)
    z = bc["X"].reshape(-1, SMALL.bottleneck_dimension)
    rng = np.random.default_rng(4)
    gam, bet = rng.standard_normal(z.shape[1]), rng.standard_normal(z.shape[1])
    eps_ln = 2.0 ** -10
    y, (xh, rstd) = STO._ln_fwd(z, gam, bet, eps_ln)
    f = R.layer_norm_forward(z, np.zeros_like(z), gam, bet, eps_ln)
    np.testing.assert_allclose(f["y"], y, rtol=0, atol=1e-12)
    np.testing.assert_allclose(f["rstd"], rstd[:, 0], rtol=0, atol=1e-12)
    dy = rng.standard_normal(z.shape)
    dz, dg, db = STO._ln_bwd(dy, gam, (xh, rstd))
    b = R.layer_norm_backward(z, np.zeros_like(z), gam, f["mean"], f["rstd"], dys=[dy])
    np.testing.assert_allclose(b["d_res"], dz, rtol=0, atol=1e-12)
    np.testing.assert_allclose(b["dgamma"][0], dg, rtol=0, atol=1e-12)
    np.testing.assert_allclose(b["dbeta"][0], db, rtol=0, atol=1e-12)


@pytest.mark.parametrize("sizes", [None, [1, 5, 70, 129]])
def test_attention_backward_agrees_with_autograd(sizes):
    S, H, L, dk = 4, 2, 6 if sizes is None else 129, 5
    q, k, v, g = (t.astype(np.float64) for t in R.attention_case(S, H, L, dk, seed=5))
    l = np.full(S, L) if sizes is None else np.asarray(sizes)
    real = torch.tensor(np.arange(L)[None, :] < l[:, None])
    tq, tk, tv = (torch.tensor(t, requires_grad=True) for t in (q, k, v))
    s = (tq / math.sqrt(dk)) @ tk.transpose(-1, -2)
    s = s.masked_fill(~real[:, None, None, :], -math.inf)
    P = torch.softmax(s, -1) * real[:, None, :, None]
    o = P @ tv
    lse = torch.logsumexp(s, -1)
    (o * torch.tensor(g)).sum().backward()
    f = R.attention_forward(q, k, v, sizes)
    np.testing.assert_allclose(f["o"], o.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(f["lse"], np.where(real[:, None].numpy(), lse.detach().numpy(), 0.0), rtol=0, atol=1e-12)
    b = R.attention_backward(q, k, v, g, f["o"], f["lse"], sizes)
    for name, t in (("dq", tq), ("dk", tk), ("dv", tv)):
        np.testing.assert_allclose(b[name], t.grad.numpy(), rtol=0, atol=1e-12, err_msg=name)


def test_layer_norm_backward_with_pooling_and_branch_agrees_with_autograd():
    rng = np.random.default_rng(6)
    S, Lmax, E = 3, 5, 36
    sizes = np.array([1, 5, 3])
    a, b = rng.standard_normal((S * Lmax, E)), np.tanh(rng.standard_normal((S * Lmax, E)))
    gam, bet = rng.standard_normal(E), rng.standard_normal(E)
    dpool, dy0 = rng.standard_normal((S, E)), rng.standard_normal((S * Lmax, E))
    ta, tb0 = torch.tensor(a, requires_grad=True), torch.tensor(np.arctanh(b), requires_grad=True)
    tg, tbe = torch.tensor(gam, requires_grad=True), torch.tensor(bet, requires_grad=True)
    z = ta + torch.tanh(tb0)
    y = torch.nn.functional.layer_norm(z, (E,), tg, tbe, eps=2.0 ** -10)
    pooled = R.pooled_dy(dpool, S * Lmax, Lmax, sizes)
    (y * torch.tensor(dy0 + pooled)).sum().backward()
    f = R.layer_norm_forward(a, b, gam, bet, 2.0 ** -10)
    np.testing.assert_allclose(f["y"], y.detach().numpy(), rtol=0, atol=1e-12)
    out = R.layer_norm_backward(a, b, gam, f["mean"], f["rstd"], dys=[dy0], pooled=pooled, branch_act="tanh", nsplit=2,
                                rows_per_split=8)
    np.testing.assert_allclose(out["d_res"], ta.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(out["d_branch"], tb0.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(out["dgamma"].sum(0), tg.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(out["dbeta"].sum(0), tbe.grad.numpy(), rtol=0, atol=1e-12)
    # the 1 / l_s weights are fl(1 / l_s) in fp32 and reach the real rows only
    assert np.all(pooled[Lmax + 5:2 * Lmax] == 0.0) and np.all(pooled[2 * Lmax + 3:] == 0.0)


@pytest.mark.parametrize("dk", [1, 4, 16, 64])
def test_dyadic_scores_are_exact_where_the_bound_says_so(dk):
    q, k, _, _ = R.attention_case(2, 2, 33, dk, "dyadic", seed=7)
    qs = (q * R.scale32(dk)).astype(np.float32)
    s, sig = R.scores(qs.astype(np.float64), k)
    assert np.all(sig == 0.0)
    part = np.zeros(s.shape, np.float32)
    for d in range(dk):                            # the kernels' fmaf chain: exact products, one rounding per step
        part = (part.astype(np.float64) + qs[..., :, None, d].astype(np.float64) * k[..., None, :, d]).astype(np.float32)
    np.testing.assert_array_equal(part.astype(np.float64), s)
    f = R.attention_forward(q[:, :, :1], k[:, :, :1], q[:, :, :1])          # L = 1: O = V, lse = s, exactly
    assert np.all(f["o_bound"] == 0.0) and np.all(f["lse_bound"] == 0.0)
    np.testing.assert_array_equal(f["o"], q[:, :, :1])


def test_normal_scores_have_nonzero_bounds():
    q, k, v, _ = R.attention_case(1, 1, 9, 12, seed=8)
    f = R.attention_forward(q, k, v)
    assert np.all(f["sigma"] > 0) and np.all(f["o_bound"] > 0) and np.all(f["lse_bound"] > 0)


@pytest.mark.parametrize("L,sizes", [(8, None), (64, None), (100, [1, 64, 32, 100]), (129, [128, 129])])
def test_pooling_is_exact_on_dyadic_rows_at_power_of_two_sizes(L, sizes):
    rng = np.random.default_rng(9)
    S = 4 if sizes is None else len(sizes)
    x = (rng.integers(-8, 9, size=(S * L, 12)) / 8.0).astype(np.float32)
    out, bnd = R.pool(x, L, sizes)
    l = np.full(S, L) if sizes is None else np.asarray(sizes)
    emul = np.zeros((S, 12), np.float32)
    for s in range(S):
        acc = np.zeros(12, np.float32)
        for p_ in range(l[s]):
            acc = acc + x[s * L + p_]
        emul[s] = acc / np.float32(l[s])
    exact = (l & (l - 1)) == 0
    assert np.all(bnd[exact] == 0.0) and np.all(bnd[~exact] > 0.0)
    np.testing.assert_array_equal(emul[exact].astype(np.float64), out[exact])
    assert np.all(np.abs(emul.astype(np.float64) - out) <= bnd)


# ---- seeded faults: each must leave at least one bound --------------------------------------------------------------------
def _breaks(mut, ref, bound):
    return bool(np.any(np.abs(np.asarray(mut) - ref) > bound))


def _softmax_o(s, v, keep):
    s = np.where(keep, s, -np.inf)
    P = np.exp(s - s.max(-1, keepdims=True))
    return (P / P.sum(-1, keepdims=True)) @ v


def test_a_dropped_key_tile_breaks_the_bound():
    q, k, v, _ = R.attention_case(1, 1, 129, 16, seed=10)
    f = R.attention_forward(q, k, v, [129])
    keep = (np.arange(129) < 64) | (np.arange(129) >= 128)
    assert _breaks(_softmax_o(f["s"], v.astype(np.float64), keep), f["o"], f["o_bound"])


def test_an_ignored_mask_breaks_the_bound():
    q, k, v, _ = R.attention_case(1, 1, 100, 12, seed=11)
    f = R.attention_forward(q, k, v, [70])
    qs = q.astype(np.float64) * float(R.scale32(12))
    o_all = _softmax_o(qs @ k[0, 0].T.astype(np.float64), v.astype(np.float64), np.ones(100, bool))
    assert _breaks(o_all[:, :, :70], f["o"][:, :, :70], f["o_bound"][:, :, :70])


def test_a_skipped_alpha_rescale_breaks_the_bound():
    q, k, v, _ = R.attention_case(1, 1, 200, 16, seed=12)
    f = R.attention_forward(q, k, v, [200])
    s, vv = f["s"][0, 0], v[0, 0].astype(np.float64)
    o, m, lsum = np.zeros((200, 16)), np.full((200, 1), -np.inf), np.zeros((200, 1))
    for k0 in range(0, 200, 64):
        st = s[:, k0:k0 + 64]
        mn = np.maximum(m, st.max(1, keepdims=True))
        p = np.exp(st - mn)
        lsum = lsum * np.exp(m - mn) + p.sum(1, keepdims=True)
        o = o + p @ vv[k0:k0 + 64]                 # o *= alpha left out
        m = mn
    assert _breaks(o / lsum, f["o"][0, 0], f["o_bound"][0, 0])


@pytest.mark.parametrize("mutate,out", [("no_D", "dq"), ("no_D", "dk"), ("no_scale", "dq")])
@pytest.mark.parametrize("sizes", [None, [50]])
def test_backward_faults_break_the_bound(mutate, out, sizes):
    q, k, v, g = R.attention_case(1, 2, 50, 12, seed=13)
    f = R.attention_forward(q, k, v, sizes)
    o32, lse32 = f["o"].astype(np.float32), f["lse"].astype(np.float32)
    ref = R.attention_backward(q, k, v, g, o32, lse32, sizes)
    mut = R.attention_backward(q, k, v, g, o32, lse32, sizes, mutate=mutate)
    assert _breaks(mut[out], ref[out], ref[out + "_bound"])


@pytest.mark.parametrize("dk,d", [(17, 16), (33, 16), (33, 32)])
def test_a_dropped_head_column_breaks_the_bound(dk, d):
    q, k, v, _ = R.attention_case(2, 1, 40, dk, seed=14)
    f = R.attention_forward(q, k, v)
    qd, vd = q.copy(), v.copy()
    qd[..., d] = 0.0                               # the score chain stops one column short ...
    assert _breaks(R.attention_forward(qd, k, v)["o"], f["o"], f["o_bound"])
    vd[..., d] = 0.0                               # ... or the output column is never formed
    assert _breaks(R.attention_forward(q, k, vd)["o"], f["o"], f["o_bound"])


@pytest.mark.parametrize("E", [8, 36, 128])
def test_layer_norm_faults_break_the_bound(E):
    rng = np.random.default_rng(15)
    a, b = rng.standard_normal((9, E)).astype(np.float32), rng.standard_normal((9, E)).astype(np.float32)
    gam, bet = rng.standard_normal(E).astype(np.float32), rng.standard_normal(E).astype(np.float32)
    f = R.layer_norm_forward(a, b, gam, bet, 1e-3)
    z = a.astype(np.float64) + b
    c = z - z.mean(1, keepdims=True)
    unbiased = c / np.sqrt((c * c).sum(1, keepdims=True) / (E - 1) + float(np.float32(1e-3))) * gam + bet
    no_eps = c / np.sqrt((c * c).mean(1, keepdims=True)) * gam + bet
    assert _breaks(unbiased, f["y"], f["y_bound"])
    assert _breaks(no_eps, f["y"], f["y_bound"])


def test_pooled_gradient_over_lmax_breaks_the_bound():
    rng = np.random.default_rng(16)
    S, Lmax, E = 3, 100, 32
    sizes = [1, 37, 100]
    a, b = rng.standard_normal((S * Lmax, E)).astype(np.float32), rng.standard_normal((S * Lmax, E)).astype(np.float32)
    gam = rng.standard_normal(E).astype(np.float32)
    dpool = rng.standard_normal((S, E)).astype(np.float32)
    f = R.layer_norm_forward(a, b, gam, gam, 1e-3)
    ref = R.layer_norm_backward(a, b, gam, f["mean"], f["rstd"], pooled=R.pooled_dy(dpool, S * Lmax, Lmax, sizes))
    mut = R.layer_norm_backward(a, b, gam, f["mean"], f["rstd"], pooled=R.pooled_dy(dpool, S * Lmax, Lmax, sizes, divide_by_lmax=True))
    assert _breaks(mut["d_res"], ref["d_res"], ref["d_res_bound"])
    assert _breaks(mut["dbeta"], ref["dbeta"], ref["dbeta_bound"])
