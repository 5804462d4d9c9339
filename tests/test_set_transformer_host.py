"""CPU: the float64 set-transformer oracle (tests/set_transformer_oracle.py) against its torch autograd twin and finite
differences, the parameter count and layout of nb-particle cell 8's shape, and SetTransformerIBNet's argument checks."""
import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests import set_transformer_oracle as STO

SMALL = STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[8], bottleneck_dimension=8, number_particles=5,
                     key_dim=4, number_heads=2, number_attention_blocks=2, ff_arch_per_block=[16, 8], final_processing_arch=[6],
                     number_positional_encoding_frequencies=3)


def small_case(seed, B=3, cfg=SMALL):
    rng = np.random.default_rng(seed)
    p = STO.init_params(cfg, rng, dtype=np.float64)
    x = rng.standard_normal((B, cfg.number_particles, cfg.particle_feature_dimensions))
    eps = rng.standard_normal((B, cfg.number_particles, cfg.bottleneck_dimension))
    y = (rng.random((B, cfg.output_dimensionality)) > 0.5).astype(np.float64)
    return p, x, y, eps


@pytest.mark.parametrize("batch_for_mean", [None, 7])
def test_oracle_gradient_matches_torch_autograd(batch_for_mean):
    p, x, y, eps = small_case(0)
    g, fr = STO.train_grads(SMALL, p, x, y, eps, 0.3, batch_for_mean=batch_for_mean)
    loss, leaf = STO.torch_loss(SMALL, p, x, y, eps, 0.3, batch_for_mean=batch_for_mean)
    loss.backward()
    gt = leaf.grad.numpy()
    off = 0
    for s in SMALL.param_shapes():                       # every variable on its own
        n = int(np.prod(s))
        np.testing.assert_allclose(g[off:off + n], gt[off:off + n], rtol=0, atol=1e-10 * max(1.0, np.abs(gt).max()))
        off += n
    if batch_for_mean is None:
        assert abs(fr.loss - loss.item()) < 1e-12


def test_oracle_gradient_matches_finite_differences():
    p, x, y, eps = small_case(1)
    g, _ = STO.train_grads(SMALL, p, x, y, eps, 0.3)
    rng = np.random.default_rng(2)
    h = 1e-6
    for i in rng.choice(p.size, 40, replace=False):
        pp, pm = p.copy(), p.copy()
        pp[i] += h
        pm[i] -= h
        fd = (STO.forward(SMALL, pp, x, eps, 0.3, y=y).loss - STO.forward(SMALL, pm, x, eps, 0.3, y=y).loss) / (2 * h)
        assert abs(fd - g[i]) < 1e-7 + 1e-5 * abs(g[i]), (i, fd, g[i])


def test_set_size_one_is_a_per_particle_network():
    """With L = 1 every softmax is over one key: attention output = V projection, the mean over particles is the identity."""
    cfg = STO.STConfig(**{**SMALL.__dict__, "number_particles": 1})
    p, x, y, eps = small_case(3, B=4, cfg=cfg)
    fr = STO.forward(cfg, p, x, eps, y=y, keep=True)
    for k in fr.cache["bc"]:
        np.testing.assert_allclose(k["P"], 1.0)


def test_parameter_count_and_layout_of_the_notebook_shape():
    import dib_b200
    cfg = STO.STConfig()                                  # nb-particle cell 8: 12 -> PE(5) -> [128, 128] -> 2*32; 6 x (12 heads, dk 128)
    E, h, dk, d = 32, 12, 128, 12
    enc = (d * 5 * 128 + 128) + (128 * 128 + 128) + (128 * 2 * E + 2 * E)
    block = 3 * (E * h * dk + h * dk) + (h * dk * E + E) + 2 * E + (E * 128 + 128) + (128 * E + E) + 2 * E
    head = (E * 256 + 256) + (256 + 1)
    assert cfg.encoder_param_count() == enc
    assert cfg.param_count() == enc + 6 * block + head
    specs = dib_b200.models.set_transformer_param_specs(d, [128, 128], E, 50, h, dk, 6, [128, E], [256], 1, 5)
    assert len(specs) == len(cfg.param_shapes())
    for (name, shape, init), s in zip(specs, cfg.param_shapes()):
        flat = tuple(shape)                               # dib_param_layout reports [E, h*dk], [h*dk] and [h*dk, E]
        if len(shape) == 3:
            flat = (shape[0] * shape[1], shape[2]) if "attention_output" in name else (shape[0], shape[1] * shape[2])
        elif len(shape) == 2 and name.endswith("bias"):
            flat = (shape[0] * shape[1],)
        assert flat == tuple(s), (name, shape, s)
    q = next(sp for sp in specs if sp[0] == "block0/query/kernel")
    o = next(sp for sp in specs if sp[0] == "block0/attention_output/kernel")
    assert q[2] == ("glorot", h * E, dk * E) and o[2] == ("glorot", dk * h, E * h)       # Keras _compute_fans of 3-D kernels


@pytest.mark.parametrize("kw, match", [
    (dict(number_particles=65), "number_particles"),
    (dict(number_particles=0), "number_particles"),
    (dict(key_dim=129), "key_dim"),
    (dict(number_heads=0), "number_heads"),
    (dict(ff_arch_per_block=[128, 16]), "last width"),
    (dict(bottleneck_dimension=30, ff_arch_per_block=[128, 30]), "multiples of 4"),
    (dict(ff_activation_fn="swish"), "activation"),
    (dict(precision="fp64"), "precision"),
])
def test_invalid_constructor_arguments_are_rejected_before_any_device_call(kw, match, monkeypatch):
    import dib_b200
    from dib_b200 import models

    def no_device(*a, **k):
        raise AssertionError("a device call was made")
    monkeypatch.setattr(models, "_require_cuda", no_device)
    monkeypatch.setattr(models._lib, "load", no_device)
    args = dict(particle_feature_dimensions=12, particle_encoder_arch_spec=[128, 128])
    with pytest.raises(ValueError, match=match):
        dib_b200.SetTransformerIBNet(**{**args, **kw})
