"""CPU: the masked float64 set-transformer oracle (tests/set_transformer_varlen_oracle.py) against its torch autograd twin, finite
differences and, at uniform sizes, the fixed-size oracle; pad_sets and the variable-size argument checks; the ABI v5 layout."""
import ctypes

import numpy as np
import pytest

from oracle import dib_oracle as O
from tests import set_transformer_oracle as STO
from tests import set_transformer_varlen_oracle as VO

SMALL = STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[8], bottleneck_dimension=8, number_particles=6,
                     key_dim=4, number_heads=2, number_attention_blocks=2, ff_arch_per_block=[16, 8], final_processing_arch=[6],
                     number_positional_encoding_frequencies=3)


def ragged_case(seed, sizes, cfg=SMALL):
    rng = np.random.default_rng(seed)
    B = len(sizes)
    p = STO.init_params(cfg, rng, dtype=np.float64)
    x = rng.standard_normal((B, cfg.number_particles, cfg.particle_feature_dimensions))
    eps = rng.standard_normal((B, cfg.number_particles, cfg.bottleneck_dimension))
    y = (rng.random((B, cfg.output_dimensionality)) > 0.5).astype(np.float64)
    return p, x, y, eps, np.asarray(sizes)


@pytest.mark.parametrize("batch_for_mean", [None, 9])
def test_masked_oracle_gradient_matches_torch_autograd(batch_for_mean):
    p, x, y, eps, sizes = ragged_case(0, [1, 6, 3, 5])
    g, fr = VO.train_grads(SMALL, p, x, y, eps, sizes, 0.3, batch_for_mean=batch_for_mean)
    loss, leaf = VO.torch_loss(SMALL, p, x, y, eps, sizes, 0.3, batch_for_mean=batch_for_mean)
    loss.backward()
    gt = leaf.grad.numpy()
    off = 0
    for s in SMALL.param_shapes():
        n = int(np.prod(s))
        np.testing.assert_allclose(g[off:off + n], gt[off:off + n], rtol=0, atol=1e-10 * max(1.0, np.abs(gt).max()))
        off += n
    if batch_for_mean is None:
        assert abs(fr.loss - loss.item()) < 1e-12


def test_masked_oracle_gradient_matches_finite_differences():
    p, x, y, eps, sizes = ragged_case(1, [2, 6, 4])
    g, _ = VO.train_grads(SMALL, p, x, y, eps, sizes, 0.3)
    rng = np.random.default_rng(2)
    h = 1e-6
    for i in rng.choice(p.size, 40, replace=False):
        pp, pm = p.copy(), p.copy()
        pp[i] += h
        pm[i] -= h
        fd = (VO.forward(SMALL, pp, x, eps, sizes, 0.3, y=y).loss - VO.forward(SMALL, pm, x, eps, sizes, 0.3, y=y).loss) / (2 * h)
        assert abs(fd - g[i]) < 1e-7 + 1e-5 * abs(g[i]), (i, fd, g[i])


def test_uniform_sizes_equal_the_fixed_size_oracle():
    p, x, y, eps, sizes = ragged_case(3, [6] * 4)
    g, fr = VO.train_grads(SMALL, p, x, y, eps, sizes, 0.2)
    g0, fr0 = STO.train_grads(SMALL, p, x, y, eps, 0.2)
    assert np.abs(g - g0).max() <= 1e-12 * max(1.0, np.abs(g0).max())
    assert abs(fr.loss - fr0.loss) < 1e-12 and abs(fr.kl - fr0.kl) < 1e-12
    assert np.abs(fr.pred - fr0.pred).max() < 1e-12


def test_each_set_is_the_fixed_size_model_at_its_own_size():
    """Per set, the masked oracle is the fixed-size oracle at L = l_s on the real particles; padding content is ignored."""
    sizes = [1, 4, 6]
    p, x, y, eps, sizes = ragged_case(4, sizes)
    x[0, 1:] = np.nan
    eps[1, 4:] = np.inf
    B = len(sizes)
    g, fr = VO.train_grads(SMALL, p, x, y, eps, sizes, 0.1)
    g_sum, kl_sum = np.zeros_like(g), 0.0
    for s, l in enumerate(sizes):
        cfg = STO.STConfig(**{**SMALL.__dict__, "number_particles": int(l)})
        gs, frs = STO.train_grads(cfg, p, x[s:s + 1, :l], y[s:s + 1], eps[s:s + 1, :l], 0.1, batch_for_mean=B)
        g_sum += gs
        kl_sum += frs.kl
        assert np.abs(fr.pred[s] - frs.pred[0]).max() < 1e-12
    assert np.isfinite(g).all()
    assert np.abs(g - g_sum).max() < 1e-12 * max(1.0, np.abs(g).max())
    assert abs(fr.kl - kl_sum / B) < 1e-12


def test_pad_sets_and_size_checks():
    from dib_b200 import models
    sets = [np.ones((2, 3)), 2 * np.ones((5, 3)), np.zeros((1, 3))]
    x, sizes = models.pad_sets(sets, 6)
    assert x.shape == (3, 6, 3) and x.dtype == np.float32 and sizes.dtype == np.int32
    assert sizes.tolist() == [2, 5, 1]
    assert (x[0, :2] == 1).all() and (x[0, 2:] == 0).all() and (x[1, :5] == 2).all() and (x[1, 5:] == 0).all()
    with pytest.raises(ValueError, match=r"\[1, 4\]"):
        models.pad_sets(sets, 4)                                         # a set larger than Lmax
    with pytest.raises(ValueError, match=r"\[1, 6\], got 0"):
        models.pad_sets([np.zeros((0, 3))], 6)                           # an empty set
    with pytest.raises(ValueError, match="every set"):
        models.pad_sets([np.zeros((2, 3)), np.zeros((2, 4))], 6)
    with pytest.raises(ValueError, match="one size per set"):
        models.check_set_sizes(np.array([1, 2]), 3, 6)                   # mismatched lengths
    with pytest.raises(ValueError, match="got 7"):
        models.check_set_sizes(np.array([1, 7, 2]), 3, 6)
    models.check_set_sizes(np.array([1, 6, 2]), 3, 6)


@pytest.mark.parametrize("kw, match", [
    (dict(number_particles=257, variable_set_sizes=True), r"\[1, 256\]"),
    (dict(number_particles=0, variable_set_sizes=True), "number_particles"),
    (dict(number_particles=65), "variable_set_sizes"),
])
def test_variable_size_constructor_checks_run_before_any_device_call(kw, match, monkeypatch):
    import dib_b200
    from dib_b200 import models

    def no_device(*a, **k):
        raise AssertionError("a device call was made")
    monkeypatch.setattr(models, "_require_cuda", no_device)
    monkeypatch.setattr(models._lib, "load", no_device)
    with pytest.raises(ValueError, match=match):
        dib_b200.SetTransformerIBNet(12, [128, 128], **kw)


def test_abi5_struct_layout():
    from dib_b200 import _lib
    assert _lib.ABI_VERSION == 5
    names = [n for n, _ in _lib.DibConfig._fields_]
    assert names[-1] == "variable_set_sizes" and names[-2] == "layer_norm_epsilon"
    assert _lib.DibConfig.variable_set_sizes.offset == _lib.DibConfig.layer_norm_epsilon.offset + 4
    assert _lib.DibConfig.variable_set_sizes.size == 4
    assert _lib.SIGNATURES["dib_set_set_sizes_device"] == (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p])
    hdr = open(__file__.replace("tests/test_set_transformer_varlen_host.py", "include/dib_b200.h")).read()
    assert "#define DIB_ABI_VERSION 5" in hdr and "#define DIB_MAX_VARIABLE_SET_SIZE 256" in hdr
    assert "int dib_set_set_sizes_device(dib_model* h, const int32_t* set_sizes_dev);" in hdr
