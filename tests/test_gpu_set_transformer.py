"""GPU (H100): SetTransformerIBNet -- nb-particle cell 8's particle encoder + set transformer as one library step -- against
the float64 oracle (tests/set_transformer_oracle.py), against itself (shards, seeds, graph replay), through fit, in tf32,
and dib_create's checks of the set-transformer fields."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import set_transformer_oracle as STO

pytestmark = pytest.mark.gpu

NOTEBOOK = STO.STConfig()            # 12 features, PE 5, [128, 128], E 32, L 50, 6 blocks of 12 heads x 128, FF [128, 32], head [256]


def small(L):
    return STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[16], bottleneck_dimension=8, number_particles=L,
                        key_dim=12, number_heads=3, number_attention_blocks=2, ff_arch_per_block=[20, 8], final_processing_arch=[12],
                        number_positional_encoding_frequencies=3)


def make_model(cfg, precision="fp32", seed=0, lr=1e-3, metrics=None):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(cfg.particle_feature_dimensions, cfg.particle_encoder_arch_spec, cfg.bottleneck_dimension,
                                     cfg.number_particles, key_dim=cfg.key_dim, number_heads=cfg.number_heads,
                                     number_attention_blocks=cfg.number_attention_blocks, ff_arch_per_block=cfg.ff_arch_per_block,
                                     final_processing_arch=cfg.final_processing_arch,
                                     number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies,
                                     precision=precision, seed=seed)
    m.compile(optimizer=dib_b200.Adam(lr), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=metrics)
    return m


def case(cfg, B, seed):
    rng = np.random.default_rng(seed)
    p = STO.init_params(cfg, rng)
    x = rng.standard_normal((B, cfg.number_particles, cfg.particle_feature_dimensions)).astype(np.float32)
    eps = rng.standard_normal((B, cfg.number_particles, cfg.bottleneck_dimension)).astype(np.float32)
    y = (rng.random((B, 1)) > 0.5).astype(np.float32)
    return p, x, y, eps


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


# per-variable bound: 2e-4 of the variable's own maximum as DESIGN section 2 at the small shapes.  At the notebook depth (6 blocks)
# the ReLU FF kernels, whose gradients are ~1 % of the flat maximum, measured up to 1.8e-3 of their own maximum (1.6e-5 absolute,
# 2e-5 of the flat maximum): there every variable is held to the flat max-norm bound instead
@pytest.mark.parametrize("cfg, B, per_var", [(NOTEBOOK, 32, None), (small(1), 16, 2e-4), (small(7), 9, 2e-4), (small(64), 5, 2e-4)],
                         ids=["notebook", "L1", "L7", "L64"])
def test_fp32_step_matches_float64_oracle(cfg, B, per_var):
    m = make_model(cfg)
    assert m.count_params() == cfg.param_count()
    assert "set_transformer=attention-simt-fp32" in m.kernel_info(B)
    p, x, y, eps = case(cfg, B, 1)
    m.set_flat_weights(p)
    m.beta.assign(0.02)
    g, st = m.compute_gradients(x, y, eps=eps)
    g, st = g.cpu().numpy(), st.cpu().numpy()
    g_ref, fr = STO.train_grads(cfg, p, x, y, eps, 0.02)
    assert rel(g, g_ref) < 5e-5                                          # max-norm over the flat gradient
    scale = np.abs(g_ref).max()
    for i in range(len(m._var_off)):                                     # and per variable
        off, n = m._var_off[i], max(m._var_rows[i], 1) * m._var_cols[i]
        # a variable whose exact gradient vanishes (the key bias: softmax ignores a per-row constant; Q and K when L = 1) is
        # measured against the flat gradient's scale: fp32 leaves rounding residue there
        ref = np.abs(g_ref[off:off + n]).max()
        bound = 5e-5 * scale if per_var is None else per_var * max(ref, 1e-3 * scale)
        assert np.abs(g[off:off + n] - g_ref[off:off + n]).max() < bound, i
    assert abs(st[0] / B - fr.kl) < 2e-5 * max(1.0, fr.kl)
    assert abs(st[1] / B - fr.task_loss) < 2e-5
    assert st[3] == B
    pred = m(x, eps=eps)
    assert np.abs(pred - fr.pred).max() < 2e-5 * max(1.0, np.abs(fr.pred).max())
    # the two callables: particle encoder (mu || logvar with the offset) and the set transformer alone
    ml = m.particle_encoder(x)
    fr2 = STO.forward(cfg, p, x, eps, keep=True)
    E = cfg.bottleneck_dimension
    ref_ml = np.concatenate([fr2.cache["mu"], fr2.cache["lv"]], -1).reshape(B, cfg.number_particles, 2 * E)
    assert rel(ml, ref_ml) < 2e-5
    u = (fr2.cache["mu"] + np.exp(fr2.cache["lv"] / 2) * eps.reshape(-1, E)).reshape(B, cfg.number_particles, E)
    assert np.abs(m.set_transformer(u.astype(np.float32)) - fr.pred).max() < 2e-5 * max(1.0, np.abs(fr.pred).max())


def test_param_layout_reports_flattened_attention_kernels():
    m = make_model(NOTEBOOK)
    shapes = NOTEBOOK.param_shapes()
    assert len(m._var_off) == len(shapes)
    for r, c, s in zip(m._var_rows, m._var_cols, shapes):
        assert ((r, c) if r else (c,)) == tuple(s)
    assert m._var_off[2 * 3] == NOTEBOOK.encoder_param_count() == 32576


def test_shards_add_up_to_the_full_batch():
    cfg, B = small(7), 12
    m = make_model(cfg)
    p, x, y, eps = case(cfg, B, 2)
    m.set_flat_weights(p)
    m.beta.assign(0.1)
    g, st = m.compute_gradients(x, y, eps=eps)
    g1, s1 = m.compute_gradients(x[:5], y[:5], eps=eps[:5], global_batch=B)
    g2, s2 = m.compute_gradients(x[5:], y[5:], eps=eps[5:], global_batch=B, sample_offset=5)
    assert rel((g1 + g2).cpu().numpy(), g.cpu().numpy()) < 1e-5
    np.testing.assert_allclose((s1 + s2).cpu().numpy(), st.cpu().numpy(), rtol=1e-5)
    # Philox noise is keyed by the global particle row: the shards draw the full batch's noise
    g, st = m.compute_gradients(x, y, step=3)
    g1, s1 = m.compute_gradients(x[:5], y[:5], global_batch=B, step=3)
    g2, s2 = m.compute_gradients(x[5:], y[5:], global_batch=B, step=3, sample_offset=5)
    assert rel((g1 + g2).cpu().numpy(), g.cpu().numpy()) < 1e-5
    np.testing.assert_allclose((s1 + s2).cpu().numpy(), st.cpu().numpy(), rtol=1e-5)


def test_seeded_runs_and_graph_replay_are_bit_identical():
    cfg, B = small(7), 16
    p, x, y, _ = case(cfg, B, 3)
    a = make_model(cfg)
    a.set_flat_weights(p)
    g1, s1 = a.compute_gradients(x, y, step=5)
    g2, s2 = a.compute_gradients(x, y, step=5)
    assert torch.equal(g1, g2) and torch.equal(s1, s2)
    runs = []
    for graph in (False, True):
        m = make_model(cfg)
        m.use_cuda_graph = graph
        m.set_flat_weights(p)
        m.beta.assign(0.05)
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        stats = [m.train_on_batch(xd, yd)["loss"] for _ in range(5)]
        assert (len(m._graphs) > 0) == graph
        runs.append((m.get_flat_weights(), stats))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert runs[0][1] == runs[1][1]


def test_fit_follows_the_oracle_history():
    import dib_b200
    cfg, B, n, nv = small(7), 8, 28, 10
    m = make_model(cfg, lr=2e-3, metrics=["accuracy"])
    m.noise_seed = 77
    p, x, y, _ = case(cfg, n + nv, 4)
    m.set_flat_weights(p)
    cb = dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)
    hist = m.fit(x[:n], y[:n], batch_size=B, epochs=3, callbacks=[cb], validation_data=(x[n:], y[n:]), verbose=0).history
    perms = {e: m.epoch_permutation(e, n).cpu().numpy() for e in range(3)}
    L, E = cfg.number_particles, cfg.bottleneck_dimension

    def eps_fn(step, set_ids):
        rows = (np.asarray(set_ids)[:, None] * L + np.arange(L)[None, :]).ravel()
        return philox.normal_noise(77, step, rows, 1, E, dtype=np.float64).reshape(len(set_ids), L, E)
    _, h_ref = STO.fit(cfg, p, x[:n].astype(np.float64), y[:n].astype(np.float64), epochs=3, batch_size=B, lr=2e-3, eps_fn=eps_fn,
                       perm_fn=lambda e, N: perms[e], beta_fn=lambda e: O.beta_schedule(e, 1e-3, 1e-1, 1, 2),
                       validation_data=(x[n:].astype(np.float64), y[n:].astype(np.float64)))
    assert set(hist) == set(h_ref)
    for k in h_ref:
        np.testing.assert_allclose(hist[k], h_ref[k], rtol=2e-3, atol=1e-6, err_msg=k)


def test_tf32_against_fp32():
    """TF32 rounds the operands of every dense layer to 10 mantissa bits (relative error <= 2^-11 ~ 4.9e-4 per operand); the
    attention core and the LayerNorms stay fp32.  Through 6 blocks at the notebook shape the measured deviation of the
    gradient from fp32 is printed; the bounds below sit above it with room (DESIGN section 2)."""
    cfg, B = NOTEBOOK, 32
    p, x, y, eps = case(cfg, B, 5)
    out = {}
    for prec in ("fp32", "tf32", "fp16"):
        m = make_model(cfg, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(0.02)
        g, st = m.compute_gradients(x, y, eps=eps)
        out[prec] = (g.cpu().numpy(), st.cpu().numpy(), m(x, eps=eps), m.kernel_info(B))
    assert "operands=tf32" in out["fp16"][3]
    eg, ep = rel(out["tf32"][0], out["fp32"][0]), np.abs(out["tf32"][2] - out["fp32"][2]).max()
    print(f"tf32 vs fp32: gradient max-norm rel {eg:.3e}, prediction abs {ep:.3e}")
    assert eg < 3e-2 and ep < 1e-2
    assert abs(out["tf32"][1][0] - out["fp32"][1][0]) < 5e-3 * abs(out["fp32"][1][0])
    assert np.array_equal(out["fp16"][0], out["tf32"][0])            # fp16 runs the TF32 kernels


def _config(**kw):
    from dib_b200 import _lib
    fd = (ctypes.c_int32 * 1)(3)
    ea = (ctypes.c_int32 * 1)(16)
    ia = (ctypes.c_int32 * 1)(12)
    ff = (ctypes.c_int32 * 2)(20, 8)
    keep = [fd, ea, ia, ff]
    base = dict(abi_version=_lib.ABI_VERSION, number_features=1, feature_dimensionalities=fd, number_encoder_layers=1,
                feature_encoder_architecture=ea, number_integration_layers=1, integration_network_architecture=ia,
                output_dimensionality=1, use_positional_encoding=1, number_positional_encoding_frequencies=3, activation_fn=3,
                leaky_relu_alpha=0.1, feature_embedding_dimension=8, output_activation_fn=0, loss=0, precision=0, max_batch=16,
                integration_kind=1, set_size=7, number_attention_blocks=2, number_heads=3, key_dim=12, number_ff_layers=2,
                ff_architecture=ff, ff_activation_fn=1)
    base.update(kw)
    return _lib.DibConfig(**base), keep


@pytest.mark.parametrize("kw, match", [
    (dict(set_size=65), "set_size"), (dict(set_size=0), "set_size"),
    (dict(number_features=2), "number_features"),
    (dict(ff_architecture=(ctypes.c_int32 * 2)(20, 12)), "last width"),
    (dict(loss=1), "loss"), (dict(loss=5), "loss"),
    (dict(dropout_rate=0.1), "dropout"),
])
def test_dib_create_rejects_bad_set_transformer_configs(kw, match):
    from dib_b200 import _lib
    lib = _lib.load()
    cfg, _ = _config(**kw)
    h = ctypes.c_void_p()
    assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
    assert match in lib.dib_last_error().decode()
    for ok in (dict(loss=4), dict(loss=2), dict(loss=3)):            # BCE on probabilities, MSE, external are accepted
        cfg, _ = _config(**ok)
        assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) == 0, lib.dib_last_error()
        lib.dib_destroy(h)


def test_abi3_struct_still_builds_an_mlp_model():
    from dib_b200 import _lib
    lib = _lib.load()

    class DibConfigV3(ctypes.Structure):
        _fields_ = _lib.DibConfig._fields_[:27]
    assert DibConfigV3._fields_[-1][0] == "infonce_temperature"
    ref, _keep = _config()
    cfg3 = DibConfigV3(**{name: getattr(ref, name) for name, _ in DibConfigV3._fields_})
    cfg3.abi_version = 3
    h = ctypes.c_void_p()
    assert lib.dib_create(ctypes.cast(ctypes.pointer(cfg3), ctypes.POINTER(_lib.DibConfig)), ctypes.byref(h)) == 0, \
        lib.dib_last_error()
    try:
        # the MLP: encoder (3*3 -> 16 -> 16) + integration 8 -> 12 -> 1, no attention parameters
        assert lib.dib_param_count(h) == (9 * 16 + 16) + (16 * 16 + 16) + (8 * 12 + 12) + (12 + 1)
    finally:
        lib.dib_destroy(h)
