"""GPU (H100): the tensor-core modes (wgmma, fp32 accumulation in registers) against the float64 oracle and the
exact-fp32 CUDA path.
  'fp16' -- fused per-feature encoder kernels + 16-bit integration path, fp16 operands (10 explicit mantissa bits,
            relative rounding 2^-11 ~ 4.9e-4, 5-bit exponent);
  'tf32' -- tf32 wgmma grouped GEMMs on fp32 storage (same mantissa, 8-bit exponent);
  'bf16' -- the fused kernels on bf16 operands (7 explicit mantissa bits, relative rounding 2^-8 ~ 3.9e-3).
Stated tolerance: with fp32 accumulation over K <= 512 terms of mixed sign the max-norm relative error of activations
and gradients stays below 5e-3 for the 11-bit-significand modes and below 4e-2 for bf16 (8x the rounding unit), which
are the bounds asserted here (the fp32 path is held to 5e-5 in test_gpu_parity)."""
import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests.test_gpu_parity import LOSS_OF, build_model, load_case, make_labels, rel_err

pytestmark = pytest.mark.gpu
TOL = 5e-3
TOLS = {"fp16": 5e-3, "tf32": 5e-3, "bf16": 4e-2}


def test_kernel_info_names_what_runs():
    """The label a handle reports is the arithmetic it runs: C0 in 'fp16' selects the fused f16 kernels, 'tf32' never
    does, an off-envelope shape in 'fp16' falls back to the tf32 kernels and says so."""
    c0 = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    assert "encoders=fused-wgmma-f16 integration=int16-wgmma-f16 operands=fp16" in build_model(c0, precision="fp16").kernel_info()
    assert "encoders=fused-wgmma-bf16 integration=int16-wgmma-bf16 operands=bf16" in build_model(c0, precision="bf16").kernel_info()
    assert "encoders=grouped-wgmma-tf32 integration=wgmma-tf32 operands=tf32" in build_model(c0, precision="tf32").kernel_info()
    assert "simt-fp32" in build_model(c0, precision="fp32").kernel_info()
    odd = O.DIBConfig([1] * 4, [64, 64], [128], 1)
    assert "encoders=grouped-wgmma-tf32" in build_model(odd, precision="fp16").kernel_info()


@pytest.mark.parametrize("prec", ["fp16", "tf32", "bf16"])
@pytest.mark.parametrize("name", ["c0_small", "radial_like", "pendulum_like", "odd_shapes"])
def test_tc_forward_and_gradients_vs_oracle(golden_dir, name, prec):
    TOL = TOLS[prec]
    cfg, z = load_case(golden_dir, name)
    loss_name, loss = LOSS_OF[name]
    m = build_model(cfg, precision=prec, loss=loss_name)
    m.set_flat_weights(z["params"])
    beta = float(z["beta"])
    m.beta.assign(beta)
    pred = m(z["x"], eps=z["eps"])
    assert rel_err(pred, z["pred"]) < TOL
    np.testing.assert_allclose(m._last_kl.cpu().numpy(), z["kl"], rtol=TOL)
    y = make_labels(np.random.default_rng(5), loss, z["x"].shape[0], cfg.output_dimensionality)
    g, stats = m.compute_gradients(z["x"], y, eps=z["eps"])
    g_ref, fr = O.train_grads(cfg, z["params"], z["x"], y, z["eps"], beta, loss)
    g = g.cpu().numpy()
    # fewer than 128 samples: single activation-sign flips under 11-bit operands are visible -> 2x the bound
    assert rel_err(g, g_ref) < (TOL if z["x"].shape[0] >= 128 else 2 * TOL)
    # per variable: with <100 samples a handful of activation-sign flips under reduced precision moves a whole
    # variable's gradient by several percent of its own (small) scale -> loose bound here, tight bound at B=4096 below
    off = 0
    for s in cfg.param_shapes():
        n = int(np.prod(s))
        assert rel_err(g[off:off + n], g_ref[off:off + n]) < (0.1 if z["x"].shape[0] >= 64 else 0.35) * (TOL / 5e-3) ** 0.5, (off, s)
        off += n


@pytest.mark.parametrize("tc", ["fp16", "tf32", "bf16"])
def test_tc_matches_fp32_path_multi_split_batch(tc):
    """4096 rows -> 16 deterministic batch splits in the weight-gradient kernels; ragged tail (4096+77)."""
    cfg = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    rng = np.random.default_rng(0)
    p = O.glorot_uniform_params(cfg, rng)
    for B in (4096, 4096 + 77):
        x = rng.standard_normal((B, 16)).astype(np.float32)
        y = (x[:, 0] * x[:, 1] > 0).astype(np.float32)[:, None]
        out = {}
        for prec in ("fp32", tc):
            m = build_model(cfg, precision=prec)
            m.set_flat_weights(p)
            m.beta.assign(0.01)
            g, st = m.compute_gradients(x, y, step=1)
            g2, st2 = m.compute_gradients(x, y, step=1)
            assert torch.equal(g, g2) and torch.equal(st, st2)          # deterministic
            out[prec] = (g.cpu().numpy(), st.cpu().numpy())
        assert rel_err(out[tc][0], out["fp32"][0]) < TOLS[tc]
        np.testing.assert_allclose(out[tc][1], out["fp32"][1], rtol=TOLS[tc])


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_tc_training_reduces_loss(prec):
    import dib_b200
    x, y = O.boolean_circuit_truth_table()
    m = dib_b200.DistributedIBNet([1] * 10, [128, 128], [256, 256], 1, precision=prec, seed=3)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
    h = m.fit(x, y, epochs=30, batch_size=256, callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-4, 1e-3, 30, 1)]).history
    assert h["loss"][-1] < 0.6 * h["loss"][0] and h["accuracy"][-1] > 0.85


@pytest.mark.parametrize("shape", ["c0", "hetero_tanh"])
def test_fused_encoder_kernels_match_unfused_and_fp32(shape):
    """The fused per-feature encoder kernels (16-bit operands, fp32 accumulate) against the unfused TF32 kernels and
    the exact fp32 path on the same inputs, incl. a ragged last tile and more rows than one wave of CTAs; the second
    shape has heterogeneous feature dimensionalities (pendulum-like [2,1,2,1]), tanh and 6 regression outputs."""
    if shape == "c0":
        cfg, loss_name, D, out = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1), "bce_logits", 16, 1
    else:
        cfg, loss_name, D, out = O.DIBConfig([2, 1, 2, 1], [128, 128], [256, 256], 6, activation_fn="tanh"), "mse", 6, 6
    rng = np.random.default_rng(3)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)      # non-zero biases
    for B in (128 * 3 + 17, 4096 + 64):
        x = rng.standard_normal((B, D)).astype(np.float32)
        y = (x[:, 0] * x[:, 1] > 0).astype(np.float32)[:, None] if out == 1 else rng.standard_normal((B, out)).astype(np.float32)
        res = {}
        for tag, prec, unfused in (("fp32", "fp32", 0), ("tc_unfused", "tf32", 0), ("tc_fused_int32", "fp16", 2),
                                   ("tc_fused", "fp16", 0)):
            m = build_model(cfg, precision=prec, loss=loss_name)
            m.debug_force_unfused(unfused)
            m.set_flat_weights(p)
            m.beta.assign(0.02)
            pred = m(x, step=5)
            g, st = m.compute_gradients(x, y, step=5)
            res[tag] = (np.asarray(pred), g.cpu().numpy(), st.cpu().numpy())
        tol_g = TOL if B >= 4096 else 4 * TOL          # a few hundred samples: sign flips of single activations show
        for tag in ("tc_unfused", "tc_fused_int32", "tc_fused"):
            assert rel_err(res[tag][0], res["fp32"][0]) < TOL, (tag, B)
            assert rel_err(res[tag][1], res["fp32"][1]) < tol_g, (tag, B)
            np.testing.assert_allclose(res[tag][2], res["fp32"][2], rtol=TOL, err_msg=f"{tag} {B}")
            off = 0
            for s in cfg.param_shapes():
                n = int(np.prod(s))
                assert rel_err(res[tag][1][off:off + n], res["fp32"][1][off:off + n]) < (10 * TOL if B >= 4096 else 0.15), (tag, B, off, s)
                off += n


@pytest.mark.parametrize("shape", ["c0", "radial3"])
def test_int16_resident_weight_gemms_match_streamed_kernels_bitwise(shape):
    """The integration FWD / DGRAD GEMMs with the weight slice resident in shared memory (BN = 128 / 256, one CTA per SM)
    issue the same MMAs in the same order as the streamed-B kernels they replace: predictions, gradients and statistics
    must be bit-identical, incl. a ragged last row tile."""
    from dib_b200 import _lib
    lib = _lib.load()
    if shape == "c0":
        cfg, D = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1), 16
    else:
        cfg, D = O.DIBConfig([1] * 12, [128, 128], [256, 256, 256], 3, activation_fn="tanh", use_positional_encoding=False), 12
    rng = np.random.default_rng(5)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    B = 128 * 37 + 19
    x = rng.standard_normal((B, D)).astype(np.float32)
    y = rng.standard_normal((B, cfg.output_dimensionality)).astype(np.float32)
    res = {}
    try:
        for rb in (0, 1):
            _lib.check(lib.dib_debug_set_variant(1, rb))
            m = build_model(cfg, precision="fp16", loss="mse")
            m.set_flat_weights(p)
            m.beta.assign(0.02)
            pred = m(x, step=2)
            g, st = m.compute_gradients(x, y, step=2)
            res[rb] = (np.asarray(pred), g.cpu().numpy(), st.cpu().numpy())
    finally:
        _lib.check(lib.dib_debug_set_variant(1, 0))
    for a, b in zip(res[0], res[1]):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("loss_name", ["bce_logits", "mse"])
def test_single_output_head_kernel_matches_generic_head(loss_name):
    """The out = 1 output-head kernel (8 rows per pass, transposing butterfly, lane-parallel loss) against the generic head:
    same arithmetic per row, a different (still fixed) summation tree for the 256-term logit -> fp32 round-off only."""
    from dib_b200 import _lib
    lib = _lib.load()
    cfg = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    rng = np.random.default_rng(6)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    B = 128 * 21 + 5
    x = rng.standard_normal((B, 16)).astype(np.float32)
    y = (x[:, :1] * x[:, 1:2] > 0).astype(np.float32) if loss_name == "bce_logits" else rng.standard_normal((B, 1)).astype(np.float32)
    res = {}
    try:
        for v in (0, 1):
            _lib.check(lib.dib_debug_set_variant(2, v))
            m = build_model(cfg, precision="fp16", loss=loss_name)
            m.set_flat_weights(p)
            m.beta.assign(0.02)
            pred = m(x, step=2)
            g, st = m.compute_gradients(x, y, step=2)
            g2, _ = m.compute_gradients(x, y, step=2)
            assert torch.equal(g, g2)                                            # deterministic
            res[v] = (np.asarray(pred), g.cpu().numpy(), st.cpu().numpy())
    finally:
        _lib.check(lib.dib_debug_set_variant(2, 1))
    assert rel_err(res[1][0], res[0][0]) < 1e-5
    assert rel_err(res[1][1], res[0][1]) < 2e-4          # the 16-bit rounding of dg can flip on a 1-ulp change of the logit
    np.testing.assert_allclose(res[1][2], res[0][2], rtol=1e-5)


@pytest.mark.parametrize("precision,act,loss_name,integ", [("fp16", "relu", "bce_logits", [256, 256]), ("bf16", "tanh", "mse", [256, 256]),
                                                        ("fp16", "tanh", "bce_logits", [128, 256, 256])])
def test_fused_integration_tail_matches_per_layer_kernels(precision, act, loss_name, integ):
    """The fused [hidden 256, hidden 256, head, loss] kernel (dib_int16_fwd2_kernel) against the per-layer GEMM kernels + head:
    the same 16-bit roundings of g1 / g2 / dg2, fp32 round-off differences only in the 256-term logit and the partial sums.
    Ragged last tile, a non-power-of-two number of tiles, a deeper integration network (one plain layer before the fused tail)."""
    from dib_b200 import _lib
    lib = _lib.load()
    cfg = O.DIBConfig([1] * 16, [128, 128], integ, 1, activation_fn=act)
    rng = np.random.default_rng(16)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    res = {}
    try:
        for B in (128 * 3 + 17, 128 * 160 + 77):
            x = rng.standard_normal((B, 16)).astype(np.float32)
            y = (x[:, :1] * x[:, 1:2] > 0).astype(np.float32) if loss_name == "bce_logits" else rng.standard_normal((B, 1)).astype(np.float32)
            for v in (0, 1):
                _lib.check(lib.dib_debug_set_variant(3, v))
                m = build_model(cfg, precision=precision, loss=loss_name)
                m.set_flat_weights(p)
                m.beta.assign(0.02)
                pred = m(x, step=2)
                g, st = m.compute_gradients(x, y, step=2)
                g2, _ = m.compute_gradients(x, y, step=2)
                assert torch.equal(g, g2)                                            # deterministic
                assert torch.isfinite(g).all()
                res[v] = (np.asarray(pred), g.cpu().numpy(), st.cpu().numpy())
            assert rel_err(res[1][0], res[0][0]) < 1e-5
            assert rel_err(res[1][1], res[0][1]) < 2e-4      # a 1-ulp change of the logit can flip a 16-bit rounding of dg2
            np.testing.assert_allclose(res[1][2], res[0][2], rtol=1e-5)
    finally:
        _lib.check(lib.dib_debug_set_variant(3, 1))
