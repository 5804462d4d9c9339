"""CPU: the rounding-aware float64 oracle of the 16-bit fused path (tests/fused16_oracle.py).
  * its rounding helper against torch's float32 -> float16 / bfloat16 conversion (round half to even, subnormals, overflow),
    and the saturating variant against the same conversion clamped to +-max;
  * with fmt=None it IS the float64 oracle: forward and gradients equal oracle/dib_oracle.py's to 1e-12;
  * with fmt='fp16' / 'bf16' it moves away from the float64 oracle by an amount of the format's order, so the roundings
    are really applied."""
import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests import fused16_oracle as Q
from tests.fp_exact import FORMATS

MAX = {"fp16": 65504.0, "bf16": float(torch.finfo(torch.bfloat16).max)}
TORCH = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _edge_values(fmt):
    t, emin, vmax = FORMATS[fmt]
    sub = 2.0 ** (emin - t + 1)                                  # smallest subnormal
    ulp1 = 2.0 ** (1 - t)                                        # quantum at 1
    v = [0.0, 1.0, 1.0 + ulp1 / 2, 1.0 + 1.5 * ulp1, 1.0 + ulp1 / 2 + 2.0 ** -23,      # ties to even, and just past a tie
         3.0 + ulp1, sub, sub / 2, 1.5 * sub, 2.5 * sub, sub * 0.49, 2.0 ** emin, 2.0 ** emin - sub,   # subnormals
         vmax, 65504.0, 65520.0, 65519.0, 70000.0, 1e5, vmax * (1 + 2.0 ** -t), 3.0e38,
         np.inf, 0.1, 1.0 / 3.0, 2.0 ** -20, 6.1e-5]
    v = np.asarray(v + [-a for a in v], dtype=np.float32)
    rng = np.random.default_rng(0)
    rnd = (rng.standard_normal(20000) * np.exp(rng.uniform(-30, 30, 20000))).astype(np.float32)
    return np.concatenate([v, rnd])


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_round_to_matches_torch_conversion(fmt):
    x = _edge_values(fmt)
    want = torch.from_numpy(x).to(TORCH[fmt]).to(torch.float64).numpy()
    got = Q.round_to(x.astype(np.float64), fmt, saturate=False)
    np.testing.assert_array_equal(got, want)
    sat = Q.round_to(x.astype(np.float64), fmt, saturate=True)
    np.testing.assert_array_equal(sat, np.clip(want, -MAX[fmt], MAX[fmt]))
    # NaN stays NaN in both variants; ties round to even
    assert np.isnan(Q.round_to(np.array([np.nan]), fmt)).all() and np.isnan(Q.round_to(np.array([np.nan]), fmt, False)).all()
    t = FORMATS[fmt][0]
    assert Q.round_to(np.array([1.0 + 2.0 ** -t]), fmt)[0] == 1.0
    assert Q.round_to(np.array([1.0 + 3 * 2.0 ** -t]), fmt)[0] == 1.0 + 2.0 ** (2 - t)


def test_round_to_fp16_edges_by_value():
    r = lambda v, s=True: float(Q.round_to(np.array([v]), "fp16", s)[0])
    assert r(65504.0) == 65504.0 and r(65519.0) == 65504.0
    assert r(65520.0, False) == np.inf and r(65520.0) == 65504.0             # the tie above max rounds to even = overflow
    assert r(2.0 ** -24) == 2.0 ** -24 and r(2.0 ** -25) == 0.0 and r(1.5 * 2.0 ** -25) == 2.0 ** -24
    assert r(-np.inf) == -65504.0 and r(-np.inf, False) == -np.inf


def _cfg(act="relu", loss=O.LOSS_BCE_LOGITS, out=1, **kw):
    out_act = "sigmoid" if loss == O.LOSS_BCE_PROBS else None
    return O.DIBConfig([1, 2, 3], [128, 128], [256, 256], out, activation_fn=act, output_activation_fn=out_act, **kw)


def _inputs(cfg, n, loss, seed=0):
    rng = np.random.default_rng(seed)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    x = rng.standard_normal((n, sum(cfg.feature_dimensionalities)))
    eps = rng.standard_normal((n, cfg.number_features, cfg.feature_embedding_dimension))
    out = cfg.output_dimensionality
    if loss == O.LOSS_SPARSE_CE_LOGITS:
        y = rng.integers(0, out, size=n).astype(np.float64)
    elif loss == O.LOSS_MSE:
        y = rng.standard_normal((n, out))
    else:
        y = rng.integers(0, 2, size=(n, out)).astype(np.float64)
    return p, x, eps, y


CASES = [("relu", O.LOSS_BCE_LOGITS, 1, {}), ("tanh", O.LOSS_MSE, 1, {}), ("leaky_relu", O.LOSS_BCE_LOGITS, 1, {}),
         ("relu", O.LOSS_SPARSE_CE_LOGITS, 3, {}), ("tanh", O.LOSS_MSE, 3, {}), ("relu", O.LOSS_BCE_PROBS, 1, {}),
         ("relu", O.LOSS_BCE_LOGITS, 1, {"logvar_offset": -3.0}), ("leaky_relu", O.LOSS_MSE, 1, {"kl_loss_exponent": 2.0})]


@pytest.mark.parametrize("act,loss,out,kw", CASES)
def test_unrounded_oracle_equals_float64_oracle(act, loss, out, kw):
    cfg = _cfg(act, loss, out, **kw)
    p, x, eps, y = _inputs(cfg, 37, loss)
    for beta in (1e-3, 1.0):
        g_ref, fr_ref = O.train_grads(cfg, p, x, y, eps, beta, loss)
        g, fr = Q.train_grads(cfg, p, x, y, eps, beta, loss, fmt=None)
        assert Q.per_variable_errors(cfg, g, g_ref).max() < 1e-12
        np.testing.assert_allclose(fr.pred, fr_ref.pred, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(fr.emb, fr_ref.emb, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(fr.kl_per_feature, fr_ref.kl_per_feature, rtol=1e-12)
        fo = Q.forward(cfg, p, x, eps, beta, y=y, loss=loss)
        fo_ref = O.forward(cfg, p, x, eps, beta, y=y, loss=loss)
        assert abs(fo.loss - fo_ref.loss) <= 1e-12 * abs(fo_ref.loss)
        np.testing.assert_allclose(fo.pred, fo_ref.pred, rtol=1e-12, atol=1e-14)


def test_unrounded_oracle_shard_and_encoder_only_step():
    """batch_for_mean (a shard of a larger batch) and the encoder-only d_emb step equal the float64 oracle's; a loss scale
    other than the default changes nothing without rounding (it is a power of two)."""
    cfg = _cfg("relu", O.LOSS_BCE_LOGITS, 1, logvar_offset=-3.0, kl_loss_exponent=2.0)
    p, x, eps, y = _inputs(cfg, 29, O.LOSS_BCE_LOGITS, seed=3)
    g_ref, _ = O.train_grads(cfg, p, x, y, eps, 0.3, O.LOSS_BCE_LOGITS, batch_for_mean=100)
    g, _ = Q.train_grads(cfg, p, x, y, eps, 0.3, O.LOSS_BCE_LOGITS, batch_for_mean=100, S=2.0 ** 20)
    assert Q.per_variable_errors(cfg, g, g_ref).max() < 1e-12
    d_emb = np.random.default_rng(4).standard_normal((29, 3 * 32)) / 29
    g_ref, _ = O.train_grads(cfg, p, x, None, eps, 0.3, "external", d_emb=d_emb)
    g, _ = Q.train_grads(cfg, p, x, None, eps, 0.3, "external", d_emb=d_emb)
    assert Q.per_variable_errors(cfg, g, g_ref).max() < 1e-12


@pytest.mark.parametrize("fmt,lo,hi", [("fp16", 1e-3, 5e-2), ("bf16", 1e-2, 3e-1)])
def test_rounded_oracle_departs_by_the_format_order(fmt, lo, hi):
    """Rounding the operands of every layer moves the gradients by a multiple of the format's unit (2^-11 fp16, 2^-8 bf16):
    at 200 rows the median over the variables of the per-variable max-norm relative distance lies in [lo, hi] (measured:
    1.5e-2 fp16, 7.6e-2 bf16 -- relu sign flips of a few rows dominate small variables), never near zero: the roundings are
    applied.  The prediction moves by about one unit."""
    cfg = _cfg("relu", O.LOSS_BCE_LOGITS, 1)
    p, x, eps, y = _inputs(cfg, 200, O.LOSS_BCE_LOGITS, seed=5)
    g_ref, fr_ref = O.train_grads(cfg, p, x, y, eps, 0.01, O.LOSS_BCE_LOGITS)
    g, fr = Q.train_grads(cfg, p, x, y, eps, 0.01, O.LOSS_BCE_LOGITS, fmt=fmt)
    med = float(np.median(Q.per_variable_errors(cfg, g, g_ref)))
    assert lo < med < hi, med
    unit = 2.0 ** -FORMATS[fmt][0]
    e = np.abs(fr.pred - fr_ref.pred).max() / np.abs(fr_ref.pred).max()
    assert unit / 50 < e < 50 * unit, e
    # emb16 is the rounded embedding, the returned emb is not
    np.testing.assert_array_equal(fr.cache["emb16"], Q.round_to(fr.emb, fmt))
    assert not np.array_equal(fr.emb, fr.cache["emb16"])
