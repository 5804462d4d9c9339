"""GPU (H100): the 16-bit fused training path ('fp16' / 'bf16': dib_enc_fused_fwd/bwd_kernel, dib_int16_fwd2_kernel with its
dgrad stages, the int16 GEMM / head kernels) against tests/fused16_oracle.py, a float64 restatement that rounds to 16 bits
exactly where the kernels round.  What is left between the two:
  * fp32 instead of float64 accumulation: ~K 2^-24 relative for K <= 512 terms, ~1e-5 at worst;
  * the SFU approximations: __sinf of the positional encoding, __expf of sigma (2^-21 relative), and for tanh the
    tanh.approx of dib_act16 (2^-11 relative -- as large as fp16's own rounding unit, see the tanh case);
  * one-ulp flips of a 16-bit rounding that these cause, and what a flip moves downstream.
With a smooth act' (tanh) that leaves 6.5e-4 (fp16) / 3.5e-3 (bf16) per variable.  With relu / leaky_relu it does not:
a one-ulp difference of a pre-activation that sits next to 0 flips the gate act'(h) of that element, which moves one row's
whole contribution to a weight-gradient column.  Measured per variable: 2.1e-2 (fp16) / 1.7e-2 (bf16) at 4 173 rows and
6.3e-2 at 127 rows, so these cases carry a bound of 0.1.  The tight checks of the relu path are the ones a gate flip cannot
reach: the statistics (3e-5), the embedding per element (2e-4 fp16), and the row-isolation tests, where every row but
the chosen ones must contribute exactly zero.  The bounds below are a few times the worst value measured on an H100 80GB
HBM3 (700 W power limit); DESIGN.md section 2 lists them.
"""
import math

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import fused16_oracle as Q
from tests.fp_exact import ulp16
from tests.gpu_cases import TOL, _c, _check, _data, _expect_route, _grad_case, _model, _params, _sms, _stats_err, rel_err

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# a. forward, per element
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_forward_per_element(prec):
    cfg = _c(F=16, act="leaky_relu")
    n = 128 * 9 + 1
    p = _params(cfg, 1)
    x, y, eps = _data(cfg, O.LOSS_BCE_LOGITS, n, 1)
    m = _model(cfg, prec, "bce_logits")
    _expect_route(m, prec, n, "dgrad")
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    xd, ed = m._to_device(x, 16), m._to_device(eps)
    pred, emb, st = m._forward(xd, None, ed, 0, 0, want_emb=True)
    pred, emb, st = (t.cpu().numpy().astype(np.float64) for t in (pred, emb, st))
    fr = Q.forward(cfg, p, x, eps, 0.01, fmt=prec)
    # emb is the unrounded u = mu + exp(logvar / 2) eps (dib_enc_fused.cu:470); per feature block, worst element reported
    worst = 0.0
    for f in range(16):
        a, b = emb[:, 32 * f:32 * f + 32], fr.emb[:, 32 * f:32 * f + 32]
        e = np.abs(a - b).max() / np.abs(b).max()
        if e > worst:
            worst, where = e, (f, np.unravel_index(np.abs(a - b).argmax(), a.shape))
    _check(f"emb/feature {prec} (worst at feature {where[0]}, row {where[1][0]})", worst, TOL[("emb", prec)])
    _check(f"pred {prec}", rel_err(pred, fr.pred), TOL[("pred", prec)])
    _check(f"KL sums {prec}", np.abs(st[:16] - fr.kl_per_feature * n).max() / np.abs(fr.kl_per_feature * n).max(), TOL[("stats", prec)])
    # the 16-bit embedding the integration network reads: r(u_kernel) and r(u_oracle) rarely differ.  Where they do, it is not
    # always by one ulp: a one-ulp flip of an h2 element upstream moves mu by 2^-11 of one term of its 128-term sum, which is
    # many ulps of a mu that is small through cancellation.  Reported: the fraction of differing elements (asserted) and the
    # largest distance in ulps of the larger term of u = mu + sigma eps (printed).
    terms = np.concatenate([np.maximum(np.abs(mu), np.abs(np.exp(lv / 2.0) * eps[:, f, :]))
                            for f, (_, _, _, mu, lv) in enumerate(fr.cache["enc"])], axis=-1)
    r_k, r_o = Q.round_to(emb, prec), Q.round_to(fr.emb, prec)
    d_ulp = np.abs(r_k - r_o) / ulp16(np.maximum(terms, np.maximum(np.abs(r_k), np.abs(r_o))), prec)
    print(f"[fused16-oracle] emb16 largest distance {prec}: {d_ulp.max():.1f} ulp of the larger term")
    _check(f"emb16 elements that differ {prec} (fraction)", np.mean(d_ulp > 0), TOL[("flip", prec)])


# ---------------------------------------------------------------------------------------------------------------------
# b. gradients and statistics, per variable
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = {
    "F16": (dict(F=16), "bce_logits", 0, "dgrad"),                               # 512-wide embedding, 4 D0 chunks
    "F12": (dict(F=12), "bce_logits", 0, "dgrad"),                               # 384 wide, 3 chunks
    "F2": (dict(F=2), "bce_logits", 0, "dgrad"),                                 # 64 wide: the smallest fused tail
    "deep": (dict(F=16, integ=(256, 256, 256)), "bce_logits", 0, "dgrad"),       # tail stops after e2, generic DGRAD below
    "head1": (dict(F=16, integ=(128, 256)), "bce_logits", 0, None),              # no fused tail: the out = 1 head kernel
    "sce3": (dict(F=16, out=3), "sparse_ce_logits", 0, None),                    # generic head
    "mse3": (dict(F=16, out=3), "mse", 0, None),
    "mask4": (dict(F=16), "bce_logits", 4, None),                                # per-layer GEMMs + head1
    "mask8": (dict(F=16), "bce_logits", 4 | 8, None),                            # ... + the generic head for out = 1
    "mask16": (dict(F=16), "bce_logits", 16, "fwd2"),                            # fused tail, separate dgrad launches
    "dims123": (dict(dims=[1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3, 1]), "bce_logits", 0, "dgrad"),   # 3 * 5 + 1 = 16
    "noPE": (dict(dims=[1, 2, 3] * 5 + [1], use_positional_encoding=False), "mse", 0, "dgrad"),
    "offset_p2": (dict(F=16, logvar_offset=-3.0, kl_loss_exponent=2.0), "bce_logits", 0, "dgrad"),
    "probs": (dict(F=12, probs=True), "bce_probs", 0, "dgrad"),
}


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_gradients_per_variable(shape, prec):
    kw, loss, mask, tail = SHAPES[shape]
    cfg = _c(**kw)
    for beta in (1e-3, 1.0):
        _grad_case(cfg, prec, loss, 128 * 32 + 77, beta, seed=3, mask=mask, tail=tail, label=shape)


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_philox_noise_step(prec):
    """In-kernel Philox noise (no eps tensor) against the oracle fed by oracle/philox.py with the same key."""
    cfg = _c(F=16)
    n = 128 * 20 + 3
    p = _params(cfg, 5)
    x, y, _ = _data(cfg, "bce_logits", n, 5)
    m = _model(cfg, prec, "bce_logits")
    _expect_route(m, prec, n, "dgrad")
    m.noise_seed = 1234
    m.set_flat_weights(p)
    m.beta.assign(0.05)
    g, st = m.compute_gradients(x, y, step=7, sample_offset=0)
    eps = philox.normal_noise(1234, 7, np.arange(n), 16, 32, dtype=np.float64)
    g_ref, fr = Q.train_grads(cfg, p, x, y, eps, 0.05, "bce_logits", fmt=prec)
    _check(f"grad/var philox {prec}", Q.per_variable_errors(cfg, g.cpu().numpy(), g_ref).max(), TOL[("grad", prec)])
    _check(f"stats philox {prec}", _stats_err(st.cpu().numpy().astype(np.float64), fr, n), TOL[("stats", prec)])


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_encoder_gradients_fp32_demb_route(prec):
    """encoder_gradients: the fp32 d_emb route of the fused encoder backward (g = d_emb * S, :619-622), KL exponent 2."""
    cfg = _c(F=16, logvar_offset=-3.0, kl_loss_exponent=2.0)
    n = 128 * 25 + 9
    p = _params(cfg, 6)
    x, _, eps = _data(cfg, "bce_logits", n, 6)
    d_emb = (np.random.default_rng(8).standard_normal((n, 512)) / n).astype(np.float32)
    m = _model(cfg, prec, "bce_logits")
    _expect_route(m, prec, n, "dgrad")
    m.set_flat_weights(p)
    for beta in (1e-3, 1.0):
        m.beta.assign(beta)
        g, st = m.encoder_gradients(x, d_emb, eps=eps)
        g_ref, fr = Q.train_grads(cfg, p, x, None, eps, beta, "external", fmt=prec, d_emb=d_emb)
        _check(f"grad/var encoder_gradients {prec} beta={beta}", Q.per_variable_errors(cfg, g.cpu().numpy(), g_ref).max(),
               TOL[("grad", prec)])


def test_tanh_approx_is_the_only_wide_gap():
    """dib_act16 evaluates tanh with tanh.approx.f32 (relative error up to ~2^-11, as large as fp16's rounding unit), which
    the oracle cannot restate: every activation then differs from the float64 tanh by up to one 16-bit ulp, on a large
    fraction of elements, not on a rare few.  Reported separately with its own bound."""
    for prec in ("fp16", "bf16"):
        _grad_case(_c(F=12, act="tanh"), prec, "mse", 128 * 32 + 77, 0.01, seed=4, label="tanh")


# ---------------------------------------------------------------------------------------------------------------------
# c. row isolation: every row but the chosen ones contributes exactly zero
# ---------------------------------------------------------------------------------------------------------------------
def _wgrad_split_rows(n, sms, F, integ):
    """Rows per batch slice of the paired int16 WGRAD launches (backward_integration in dib_api.cu): the slice boundaries."""
    dims = [F * 32] + list(integ)
    tiles = lambda j: math.ceil(dims[j] / 128) * math.ceil(dims[j + 1] / 128)
    part_rows = max(math.ceil(sms / F), 32)
    out, j = [], len(integ) - 1
    while j >= 1:
        ns = max(min((2 * sms) // (tiles(j) + tiles(j - 1)), part_rows, n // 256), 1)
        out.append(math.ceil(math.ceil(n / ns) / 64) * 64)
        j -= 2
    return out


def _chosen_rows(n, sms, F, integ):
    tiles = math.ceil(n / 128)
    rows = {0, n - 1, 127, 128, 128 * (tiles - 1), min(128 * (tiles - 1) + 1, n - 1)}
    for rps in _wgrad_split_rows(n, sms, F, integ):
        for b in (rps, 2 * rps, rps * ((n - 1) // rps)):
            rows |= {b - 1, b}
    # a tile served by a feature's extra CTA slot of the fused encoder backward (features f < G % F own ceil(G / F) slots)
    G = min(F * tiles, sms)
    if G >= F and G % F:
        slots_max = math.ceil(G / F)
        rows |= {128 * (slots_max - 1) + 5, 128 * (2 * slots_max - 1) + 77}
    return np.array(sorted(r for r in rows if 0 <= r < n))


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_row_isolation_training_step(prec):
    """MSE with a linear output and beta = 0, y set to the kernel's own forward-only prediction: the MSE gradient 2 (z - t)
    (dib_common.cuh:62) is exactly 0 on every row, so the step is exactly zero.  Then y moves on chosen rows only -- both
    sides of every weight-gradient slice boundary, the ragged tile's first and last row, rows 127 / 128, a tile of a
    feature's extra CTA slot -- and the step must be those rows' contribution alone, as the oracle computes it on them."""
    sms = _sms()
    cfg = _c(F=16)
    n = 20557                      # 161 tiles, ragged last tile of 77 rows; 132 SMs: 4 features get 9 backward CTA slots
    p = _params(cfg, 9)
    x, _, eps = _data(cfg, "mse", n, 9)
    m = _model(cfg, prec, "mse")
    _expect_route(m, prec, n, "dgrad")
    m.set_flat_weights(p)
    m.beta.assign(0.0)
    y = np.asarray(m(x, eps=eps), dtype=np.float32)
    g0, st0 = m.compute_gradients(x, y, eps=eps)
    # the training forward reproduces the forward-only prediction bit for bit: no row has a loss or a gradient
    assert float(st0[16]) == 0.0, ("training and forward-only predictions differ", float(st0[16]))
    assert int(torch.count_nonzero(g0)) == 0, int(torch.count_nonzero(g0))
    rows = _chosen_rows(n, sms, 16, cfg.integration_network_architecture)
    y1 = y.copy()
    y1[rows] += np.where(np.arange(len(rows)) % 2 == 0, 0.25, -0.375).astype(np.float32)[:, None]
    g, st = m.compute_gradients(x, y1, eps=eps)
    g, st = g.cpu().numpy().astype(np.float64), st.cpu().numpy().astype(np.float64)
    want_loss = float(np.sum((y[rows].astype(np.float64) - y1[rows]) ** 2))
    _check(f"row-isolation loss statistic {prec}", abs(st[16] - want_loss) / want_loss, 1e-6)
    g_ref, _ = Q.train_grads(cfg, p, x[rows], y1[rows], eps[rows], 0.0, "mse", fmt=prec, batch_for_mean=n)
    pv = Q.per_variable_errors(cfg, g, g_ref)
    _check(f"grad/var row isolation {prec} ({len(rows)} rows, worst var {int(pv.argmax())})", pv.max(), TOL[("rowiso", prec)])


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_row_isolation_encoder_gradients(prec):
    """encoder_gradients with d_emb non-zero on the chosen rows only and beta = 0."""
    sms = _sms()
    cfg = _c(F=16)
    n = 20557
    p = _params(cfg, 10)
    x, _, eps = _data(cfg, "bce_logits", n, 10)
    rows = _chosen_rows(n, sms, 16, cfg.integration_network_architecture)
    d_emb = np.zeros((n, 512), np.float32)
    d_emb[rows] = (np.random.default_rng(11).standard_normal((len(rows), 512)) / n).astype(np.float32)
    m = _model(cfg, prec, "bce_logits")
    _expect_route(m, prec, n, "dgrad")
    m.set_flat_weights(p)
    m.beta.assign(0.0)
    g, _ = m.encoder_gradients(x, d_emb, eps=eps)
    g_ref, _ = Q.train_grads(cfg, p, x[rows], None, eps[rows], 0.0, "external", fmt=prec, batch_for_mean=n, d_emb=d_emb[rows])
    pv = Q.per_variable_errors(cfg, g.cpu().numpy(), g_ref)
    _check(f"grad/var row isolation encoder_gradients {prec}", pv.max(), TOL[("rowiso", prec)])


# ---------------------------------------------------------------------------------------------------------------------
# d. scheduling edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 127, 128, 129, 128 * 9 + 1, 1024, 1025])
def test_batch_size_edges(n):
    """Single row, one ragged tile, exactly one tile, one row into the second tile, nine tiles + 1; B = 1024 / 1025 where the
    loss scale doubles (S = 1024 -> 2048)."""
    for prec in ("fp16", "bf16"):
        _grad_case(_c(F=16), prec, "bce_logits", n, 0.05, seed=12, label="edge")


@pytest.mark.parametrize("F", [2, 12, 16])
def test_encoder_schedule_around_sm_count(F):
    """F * ceil(n / 128) just below, at (when F divides it) and just above the SM count: backward_encoders launches
    min(F * tiles, SMs) CTAs, so the schedule moves from one tile per CTA to several; F = 16 does not divide 132, so
    some features own one CTA slot more than others (the slots_max != slots_min memset path)."""
    sms = _sms()
    t_eq = sms // F
    for tiles in sorted({t_eq, t_eq + 1} | ({t_eq - 1} if sms % F == 0 else set())):
        n = 128 * tiles - 37
        _grad_case(_c(F=F), "fp16", "bce_logits", n, 0.05, seed=13, label=f"sched F={F} tiles={tiles}")


def test_subnormal_gradient_operands():
    """beta ~ 1e-6 and |d_emb| ~ 1e-9: the S-scaled 16-bit gradient operands sit in fp16's subnormal range (< 6.1e-5),
    which the oracle rounds exactly (quantum 2^-24)."""
    cfg = _c(F=16)
    n = 4096
    _grad_case(cfg, "fp16", "bce_logits", n, 1e-6, seed=14, label="tiny-beta")
    p = _params(cfg, 15)
    x, _, eps = _data(cfg, "bce_logits", n, 15)
    d_emb = (np.random.default_rng(16).standard_normal((n, 512)) * 1e-9).astype(np.float32)
    m = _model(cfg, "fp16", "bce_logits")
    m.set_flat_weights(p)
    m.beta.assign(1e-6)
    g, _ = m.encoder_gradients(x, d_emb, eps=eps)
    g_ref, _ = Q.train_grads(cfg, p, x, None, eps, 1e-6, "external", fmt="fp16", d_emb=d_emb)
    assert np.abs(d_emb * Q.loss_scale(n)).max() < 2.0 ** -14                 # the operands really are subnormal
    _check("grad/var subnormal d_emb fp16", Q.per_variable_errors(cfg, g.cpu().numpy(), g_ref).max(), TOL[("grad", "fp16")])


# ---------------------------------------------------------------------------------------------------------------------
# the packing conversions saturate like the activations
# ---------------------------------------------------------------------------------------------------------------------
def test_weight_beyond_fp16_range_saturates():
    """A weight of 1e5 (beyond fp16's 65 504) in an encoder layer and in the integration network packs as 65 504
    (cvt.rn.satfinite, as every activation operand), so the fp16 step is finite and equals the oracle with saturated
    weights; a non-saturating conversion made it inf and the step NaN.  The encoder weight feeds a mu output: on the
    log-variance half it would make exp(logvar / 2) overflow in any arithmetic."""
    cfg = _c(F=16)
    p = _params(cfg, 17)
    encs, integ = O.unflatten(cfg, p)                                           # views into p
    encs[0][2][0][3, 5] = 1e5
    integ[0][0][7, 11] = -1e5
    _grad_case(cfg, "fp16", "bce_logits", 128 * 12 + 5, 0.05, seed=17, p=p, label="weight 1e5")


# ---------------------------------------------------------------------------------------------------------------------
# sparse labels outside [0, C): one rule on every loss kernel (dib_sparse_label)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("out,mask", [(3, 0), (1, 0), (1, 4)])
def test_out_of_range_sparse_label_gives_nan_loss_and_gradient(prec, out, mask):
    """An invalid label (here C, or NaN) makes the row's loss and d loss / d z NaN, as TensorFlow on a GPU does; the accuracy
    slot stays finite.  out = 3: the generic head; out = 1: the fused tail (mask 0) or the out = 1 head kernel (mask 4).
    The same batch with its labels in range stays finite."""
    if prec == "fp32" and mask:
        pytest.skip("the fp32 path has one loss kernel")
    cfg = _c(F=4, out=out)
    n = 300
    x, y, eps = _data(cfg, O.LOSS_SPARSE_CE_LOGITS, n, seed=5)
    m = _model(cfg, prec, "sparse_ce_logits", mask=mask)
    m.set_flat_weights(_params(cfg, 5))
    g, st = (t.cpu().numpy() for t in m.compute_gradients(x, y, eps=eps))
    assert np.isfinite(g).all() and np.isfinite(st).all()
    F = cfg.number_features
    for bad in (float(out), np.nan, -1.0):
        yb = y.copy()
        yb[17] = bad
        g, st = (t.cpu().numpy() for t in m.compute_gradients(x, yb, eps=eps))
        assert np.isnan(st[F]), (bad, st[F])
        assert np.isfinite(st[F + 1]) and np.isfinite(st[:F]).all(), st
        assert np.isnan(g).any(), bad
