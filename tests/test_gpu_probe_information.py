"""GPU (H100): per-probe information maps (dib_mi_bounds_at_probes, utils.estimate_mi_bounds_at_probes) and the set
information of utils.estimate_set_information / ParticleInformationCallback, against the float64 oracle
(tests/probe_information_oracle.py), against themselves (repeats, probe subsets, padding) and against the training run
they must leave untouched."""

import numpy as np
import pytest
import torch

from oracle import philox
from tests import probe_information_oracle as PO
from tests import set_transformer_oracle as STO

pytestmark = pytest.mark.gpu


def _ml(rng, n, E, mu_scale=1.0, lv_lo=-1.0, lv_hi=0.5):
    return np.concatenate([mu_scale * rng.standard_normal((n, E)), rng.uniform(lv_lo, lv_hi, (n, E))], 1).astype(np.float32)


def _run(P, D, sizes, eps=None, seed=0):
    from dib_b200 import utils
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    e = None if eps is None else torch.from_numpy(eps).cuda()
    return utils.mi_bounds_at_probes(torch.from_numpy(P).cuda(), torch.from_numpy(D).cuda(), off, e, seed).cpu().numpy()


def _oracle(P, D, sizes, eps):
    E = P.shape[1] // 2
    off = np.concatenate([[0], np.cumsum(sizes)])
    dm = [D[off[b]:off[b + 1], :E] for b in range(len(sizes))]
    dl = [D[off[b]:off[b + 1], E:] for b in range(len(sizes))]
    return PO.mi_bounds_at_probes(P[:, :E], P[:, E:], dm, dl, eps)


@pytest.mark.parametrize("E", [1, 5, 32, 64, 128])
@pytest.mark.parametrize("M", [1, 127, 1000])
def test_kernel_matches_oracle_with_explicit_noise(E, M):
    rng = np.random.default_rng(E * 1000 + M)
    sizes = [1, 63, 2048, 17]
    P, D = _ml(rng, M, E), _ml(rng, sum(sizes), E)
    eps = rng.standard_normal((len(sizes), M, E)).astype(np.float32)
    got = _run(P, D, sizes, eps)
    assert np.abs(got - _oracle(P, D, sizes, eps)).max() < 1e-9


def test_kernel_range_edges():
    rng = np.random.default_rng(5)
    E, M, sizes = 32, 200, [300, 40]
    P, D = _ml(rng, M, E, 25.0, -8.0, 2.0), _ml(rng, sum(sizes), E, 25.0, -8.0, 2.0)
    P[:, :E] = np.clip(P[:, :E], -50, 50)
    D[:, :E] = np.clip(D[:, :E], -50, 50)
    D[:20] = P[:20]                               # some rows sit on their probes: finite, informative log densities
    eps = rng.standard_normal((len(sizes), M, E)).astype(np.float32)
    got = _run(P, D, sizes, eps)
    ref = _oracle(P, D, sizes, eps)
    assert np.all(np.isfinite(got))
    assert np.abs(got - ref).max() < 1e-6


def test_philox_noise_repeats_and_probe_subsets():
    rng = np.random.default_rng(6)
    E, M, sizes, seed = 32, 300, [500, 77, 1000], 1234
    P, D = _ml(rng, M, E), _ml(rng, sum(sizes), E)
    got = _run(P, D, sizes, None, seed)
    eps = np.stack([philox.normal_noise(seed, b, np.arange(M), 1, E, dtype=np.float64)[:, 0] for b in range(len(sizes))])
    assert np.abs(got - _oracle(P, D, sizes, eps)).max() < 1e-4
    assert np.array_equal(got, _run(P, D, sizes, None, seed))
    sub = _run(P[:1], D, sizes, None, seed)       # probe 0 alone has the same key, hence the same bits
    assert np.array_equal(sub[0], got[0])


def test_notebook_shape_in_one_call():
    rng = np.random.default_rng(7)
    E, M, B, N = 32, 10000, 16, 25600
    P, D = _ml(rng, M, E), _ml(rng, B * N, E)
    got = _run(P, D, [N] * B, None, 9)
    pick = rng.choice(M, 64, replace=False)
    eps = np.stack([philox.normal_noise(9, b, pick, 1, E, dtype=np.float64)[:, 0] for b in range(B)])
    assert np.abs(got[pick] - _oracle(P[pick], D, [N] * B, eps)).max() < 1e-4


# ---------------------------------------------------------------------------------------------------- SetTransformerIBNet
def small(L):
    return STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[16], bottleneck_dimension=8, number_particles=L,
                        key_dim=12, number_heads=3, number_attention_blocks=2, ff_arch_per_block=[20, 8], final_processing_arch=[12],
                        number_positional_encoding_frequencies=3)


def make_model(cfg, variable=False, seed=0):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(cfg.particle_feature_dimensions, cfg.particle_encoder_arch_spec, cfg.bottleneck_dimension,
                                     cfg.number_particles, key_dim=cfg.key_dim, number_heads=cfg.number_heads,
                                     number_attention_blocks=cfg.number_attention_blocks, ff_arch_per_block=cfg.ff_arch_per_block,
                                     final_processing_arch=cfg.final_processing_arch,
                                     number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies,
                                     seed=seed, variable_set_sizes=variable)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True))
    return m


@pytest.mark.parametrize("cfg", [small(7), STO.STConfig()], ids=["small", "notebook"])
def test_set_transformer_probe_map_matches_oracle(cfg):
    from dib_b200 import utils
    rng = np.random.default_rng(8)
    N, M, bs, nb, seed = 40, 50, 12, 3, 21
    L, d, E = cfg.number_particles, cfg.particle_feature_dimensions, cfg.bottleneck_dimension
    m = make_model(cfg)
    x = rng.standard_normal((N, L, d)).astype(np.float32)
    probes = rng.standard_normal((M, d)).astype(np.float32)
    got = utils.estimate_mi_bounds_at_probes(m.particle_encoder, probes, x, bs, nb, seed)
    idx = utils.draw_evaluation_batches(N, bs, nb, seed, m.device).cpu().numpy()
    enc_p = np.asarray(m.particle_encoder(probes), np.float64)
    enc_x = np.asarray(m.particle_encoder(x), np.float64)
    dm = [enc_x[idx[b]].reshape(-1, 2 * E)[:, :E] for b in range(nb)]
    dl = [enc_x[idx[b]].reshape(-1, 2 * E)[:, E:] for b in range(nb)]
    eps = np.stack([philox.normal_noise(seed, b, np.arange(M), 1, E, dtype=np.float64)[:, 0] for b in range(nb)])
    ref = PO.mi_bounds_at_probes(enc_p[:, :E], enc_p[:, E:], dm, dl, eps)
    assert np.abs(got - ref).max() < 1e-4


def test_variable_model_uniform_sizes_and_nan_padding():
    from dib_b200 import utils
    cfg = small(7)
    rng = np.random.default_rng(9)
    N, M, L, d = 30, 20, 7, 3
    fixed, var = make_model(cfg), make_model(cfg, variable=True)
    var.set_flat_weights(fixed.get_flat_weights())
    x = rng.standard_normal((N, L, d)).astype(np.float32)
    probes = rng.standard_normal((M, d)).astype(np.float32)
    a = utils.estimate_mi_bounds_at_probes(fixed.particle_encoder, probes, x, 8, 4, 3)
    b = utils.estimate_mi_bounds_at_probes(var.particle_encoder, probes, (x, np.full(N, L, np.int32)), 8, 4, 3)
    assert np.array_equal(a, b)
    sizes = rng.integers(1, L + 1, N).astype(np.int32)
    xz, xn = x.copy(), x.copy()
    for i, s in enumerate(sizes):
        xz[i, s:] = 0.0
        xn[i, s:] = np.nan
    z = utils.estimate_mi_bounds_at_probes(var.particle_encoder, probes, (xz, sizes), 8, 4, 3)
    n = utils.estimate_mi_bounds_at_probes(var.particle_encoder, probes, (xn, sizes), 8, 4, 3)
    assert np.all(np.isfinite(z)) and np.array_equal(z, n)


def test_probe_call_leaves_the_training_state_untouched():
    from dib_b200 import utils
    cfg = small(7)
    rng = np.random.default_rng(10)
    m = make_model(cfg)
    x = torch.from_numpy(rng.standard_normal((32, 7, 3)).astype(np.float32)).cuda()
    y = torch.from_numpy((rng.random((32, 1)) > 0.5).astype(np.float32)).cuda()
    for _ in range(4):
        m.train_on_batch(x, y)
    assert len(m._graphs) > 0
    state = (m._max_batch, m._workspace.data_ptr(), dict(m._graphs), m._train_step_count, m._inference_calls)
    big = rng.standard_normal((600, 7, 3)).astype(np.float32)
    utils.estimate_mi_bounds_at_probes(m.particle_encoder, rng.standard_normal((10, 3)).astype(np.float32), big, 512, 2)
    utils.estimate_set_information(m, big, 512, 2)
    assert (m._max_batch, m._workspace.data_ptr(), m._train_step_count, m._inference_calls) == \
        (state[0], state[1], state[3], state[4])
    assert m._graphs.keys() == state[2].keys() and all(m._graphs[k] is state[2][k] for k in state[2])


def test_fit_with_the_callback_is_bit_identical(tmp_path):
    import dib_b200
    cfg = small(7)
    rng = np.random.default_rng(11)
    x = rng.standard_normal((40, 7, 3)).astype(np.float32)
    y = (rng.random((40, 1)) > 0.5).astype(np.float32)
    probes = rng.standard_normal((15, 3)).astype(np.float32)
    runs = []
    for with_cb in (False, True):
        m = make_model(cfg, seed=4)
        m.noise_seed = 5
        cbs = [dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)]
        if with_cb:
            pic = dib_b200.ParticleInformationCallback(1, x[32:], probes, evaluation_batch_size=4, number_evaluation_batches=2,
                                                       probe_evaluation_batch_size=8, probe_number_evaluation_batches=2,
                                                       outdir=str(tmp_path))
            cbs.append(pic)
        h = m.fit(x[:32], y[:32], batch_size=8, epochs=3, callbacks=cbs, validation_data=(x[32:], y[32:]), verbose=0).history
        runs.append((h, m.get_flat_weights()))
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1])
    assert len(pic.bounds) == 3 and len(pic.probe_bounds) == 3
    for rec in pic.probe_bounds:
        f = tmp_path / f"probe_information_log10beta_{np.log10(rec['beta']):.3f}.npz"
        z = np.load(f)
        assert set(z.files) == {"epoch", "beta", "bounds"} and z["bounds"].shape == (15, 2)


def test_set_information_is_L_times_the_batched_kernel():
    import ctypes
    from dib_b200 import _lib, utils
    cfg = small(7)
    rng = np.random.default_rng(12)
    m = make_model(cfg)
    N, bs, nb, seed, L, E = 50, 6, 3, 2, 7, 8
    x = rng.standard_normal((N, L, 3)).astype(np.float32)
    got = utils.estimate_set_information(m, x, bs, nb, seed)
    idx = utils.draw_evaluation_batches(N, bs, nb, seed, m.device)
    ml = m.particle_encoder(torch.from_numpy(x).cuda())[idx].reshape(nb, bs * L, 2 * E).contiguous()
    scratch = torch.empty(nb * bs * L * 2, dtype=torch.float64, device="cuda")
    out = torch.empty(nb, 2, dtype=torch.float64, device="cuda")
    _lib.check(_lib.load().dib_mi_sandwich_bounds_batched(_lib.ptr(ml), nb, bs * L, E, None, seed, nb, _lib.ptr(scratch),
                                                          _lib.ptr(out), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert np.allclose(got, L * out.mean(0).cpu().numpy(), rtol=0, atol=1e-12)
    # and against the float64 sandwich oracle with the same Philox noise
    from oracle import dib_oracle as O
    mlh = ml.double().cpu().numpy()
    ref = [O.mi_sandwich_batch(mlh[b, :, :E], mlh[b, :, E:],
                               philox.normal_noise(seed << 8, b, np.arange(bs * L), 1, E, dtype=np.float64)[:, 0])
           for b in range(nb)]
    assert np.abs(got - L * np.mean(ref, 0)).max() < 1e-3


def test_feature_encoder_known_answer_on_the_boolean_circuit():
    import dib_b200
    from dib_b200 import utils
    m = dib_b200.DistributedIBNet([1] * 3, "simple", [8], 1, feature_embedding_dimension=1, seed=0)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True))
    w = m.get_flat_weights()
    w[:6] = np.tile([200.0, -10.0], 3).astype(np.float32)      # (mu_scaling, logvar) per feature: mu = +-200, sigma = e^-5
    m.set_flat_weights(w)
    rng = np.random.default_rng(13)
    x = np.where(rng.random((300, 3)) > 0.3, 1.0, -1.0).astype(np.float32)
    bs, nb, seed = 40, 4, 8
    got = utils.estimate_mi_bounds_at_probes(m.feature_encoders[1], np.array([[1.0], [-1.0]], np.float32), x[:, 1:2], bs,
                                             nb, seed)
    idx = utils.draw_evaluation_batches(300, bs, nb, seed, m.device).cpu().numpy()
    ref = np.zeros((2, 2))
    for b in range(nb):
        v = x[idx[b], 1]
        for i, s in enumerate((1.0, -1.0)):
            k = int((v == s).sum())
            ref[i] += [np.log((bs + 1) / (k + 1)), np.log(bs / k) if k else np.nan]
    ref /= nb
    assert np.abs(got[:, 0] - ref[:, 0]).max() < 1e-6
    ok = np.isfinite(ref[:, 1])
    assert np.abs(got[ok, 1] - ref[ok, 1]).max() < 1e-6
