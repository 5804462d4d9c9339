"""GPU (H100): the fused encoder kernels' walking schedule against tests/fused16_oracle.py.

With fewer CTAs than features (backward_encoders launches min(F * tiles, SMs) CTAs), sched_of in dib_enc_fused.cu hands
CTA c the features c, c + G, ... with all of their tiles, so one CTA reloads the encoder weights for several features and
carries its tile sequence (the [pe|1] buffer parity, the d_emb16 load phase) across features.  The other fused16 tests use
F <= 16, which never reaches that path.  F = 140 scalar features at five tiles (the last ragged) do, for both noise routes
(explicit eps, in-kernel Philox) and both gradient routes into the encoder backward (the 16-bit d_emb16 of the fused
training step, the fp32 d_emb of encoder_gradients).  Bounds are those of test_gpu_fused16_vs_rounding_oracle.py, except
the per-variable gradient bound in bf16: with relu, a one-ulp difference next to 0 flips act' and moves one row's whole
contribution (see that module's notes), and at 583 rows over 140 features the worst variable measured 1.3e-1 in bf16
(fp16: 3.9e-2) on an H100 80GB HBM3, 700 W.  A schedule error (a wrong feature, tile or weight set) moves every variable
of a feature by O(1), and the KL and loss sums keep their 3e-5 bound.
"""
import numpy as np
import pytest

from oracle import philox
from tests import fused16_oracle as Q
from tests.gpu_cases import FUSED, TOL, _c, _check, _data, _model, _params, _sms, _stats_err

pytestmark = pytest.mark.gpu

F = 140
N = 128 * 4 + 71          # five tiles per feature; the last is ragged
SEED, STEP = 4321, 3
GRAD_TOL = {"fp16": TOL[("grad", "fp16")], "bf16": 0.25}


def _walking_model(prec, seed):
    cfg = _c(F=F)
    m = _model(cfg, prec, "bce_logits")
    info = m.kernel_info(N)
    assert FUSED[prec].split()[0] in info, info                  # encoders=fused-wgmma-*: the fused encoder kernels
    assert F > _sms(), "the walking schedule needs more features than SMs"
    p = _params(cfg, seed)
    m.set_flat_weights(p)
    return cfg, m, p


def _philox_eps():
    return philox.normal_noise(SEED, STEP, np.arange(N), F, 32, dtype=np.float64)


@pytest.mark.parametrize("noise", ["eps", "philox"])
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_walking_schedule_training_step(prec, noise):
    """compute_gradients: the fused training step, whose encoder backward reads the 16-bit d_emb16."""
    cfg, m, p = _walking_model(prec, 21)
    x, y, eps = _data(cfg, "bce_logits", N, 21)
    m.beta.assign(0.05)
    if noise == "eps":
        g, st = m.compute_gradients(x, y, eps=eps)
    else:
        m.noise_seed = SEED
        g, st = m.compute_gradients(x, y, step=STEP, sample_offset=0)
        eps = _philox_eps()
    g_ref, fr = Q.train_grads(cfg, p, x, y, eps, 0.05, "bce_logits", fmt=prec)
    g, st = g.cpu().numpy().astype(np.float64), st.cpu().numpy().astype(np.float64)
    assert np.isfinite(g).all() and np.isfinite(st).all()
    _check(f"grad/var walking {prec} {noise}", Q.per_variable_errors(cfg, g, g_ref).max(), GRAD_TOL[prec])
    _check(f"stats walking {prec} {noise}", _stats_err(st, fr, N), TOL[("stats", prec)])


@pytest.mark.parametrize("noise", ["eps", "philox"])
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_walking_schedule_encoder_gradients(prec, noise):
    """encoder_gradients: the encoder backward alone, on the fp32 d_emb route."""
    cfg, m, p = _walking_model(prec, 22)
    x, _, eps = _data(cfg, "bce_logits", N, 22)
    d_emb = (np.random.default_rng(23).standard_normal((N, F * 32)) / N).astype(np.float32)
    m.beta.assign(0.05)
    if noise == "eps":
        g, _ = m.encoder_gradients(x, d_emb, eps=eps)
    else:
        m.noise_seed = SEED
        g, _ = m.encoder_gradients(x, d_emb, step=STEP, sample_offset=0)
        eps = _philox_eps()
    g_ref, _ = Q.train_grads(cfg, p, x, None, eps, 0.05, "external", fmt=prec, d_emb=d_emb)
    g = g.cpu().numpy().astype(np.float64)
    assert np.isfinite(g).all()
    _check(f"grad/var walking encoder_gradients {prec} {noise}", Q.per_variable_errors(cfg, g, g_ref).max(),
           GRAD_TOL[prec])
