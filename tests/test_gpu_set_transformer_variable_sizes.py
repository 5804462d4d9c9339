"""GPU (H100): SetTransformerIBNet(variable_set_sizes=True) -- sets of different sizes padded to number_particles, masked
attention and pooling on the key-tiled kernels -- against the masked float64 oracle (tests/set_transformer_varlen_oracle.py),
against the fixed-size model at each set's size, against itself (padding content, shards, seeds, graph replay with changing
sizes), through fit on a ragged list, in tf32, and dib_create's limits."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import set_transformer_oracle as STO
from tests import set_transformer_varlen_oracle as VO
from tests.gpu_cases import _config, rel_err, set_transformer_model, small, varlen_set_case

pytestmark = pytest.mark.gpu

NOTEBOOK100 = STO.STConfig(number_particles=100)     # nb-particle cell 8's network on neighbourhoods of up to 100 particles


def _sizes(lo, hi, B, seed):
    return np.random.default_rng(seed).integers(lo, hi + 1, B).astype(np.int32)


CASES = [(NOTEBOOK100, _sizes(20, 100, 24, 0), None),
         (small(1), np.ones(6, np.int32), 2e-4),
         (small(7), np.array([1, 7, 3, 7, 5, 1, 2, 6, 4], np.int32), 2e-4),
         (small(65), np.array([1, 65, 64, 33, 2], np.int32), 2e-4),
         (small(256), np.array([1, 256, 129, 64, 200], np.int32), 2e-4)]


@pytest.mark.parametrize("cfg, sizes, per_var", CASES, ids=["notebook-Lmax100", "Lmax1", "Lmax7", "Lmax65", "Lmax256"])
def test_fp32_step_matches_masked_float64_oracle(cfg, sizes, per_var):
    B = len(sizes)
    m = set_transformer_model(cfg, variable=True)
    assert "set_transformer=attention-varlen-simt-fp32" in m.kernel_info(B)
    p, x, y, eps, sizes = varlen_set_case(cfg, sizes, 1)
    m.set_flat_weights(p)
    m.beta.assign(0.02)
    g, st = m.compute_gradients((x, sizes), y, eps=eps)
    g, st = g.cpu().numpy(), st.cpu().numpy()
    g_ref, fr = VO.train_grads(cfg, p, x, y, eps, sizes, 0.02)
    assert rel_err(g, g_ref) < 5e-5
    scale = np.abs(g_ref).max()
    for i in range(len(m._var_off)):
        off, n = m._var_off[i], max(m._var_rows[i], 1) * m._var_cols[i]
        ref = np.abs(g_ref[off:off + n]).max()
        bound = 5e-5 * scale if per_var is None else per_var * max(ref, 1e-3 * scale)
        assert np.abs(g[off:off + n] - g_ref[off:off + n]).max() < bound, i
    assert abs(st[0] / B - fr.kl) < 2e-5 * max(1.0, fr.kl)
    assert abs(st[1] / B - fr.task_loss) < 2e-5
    assert st[3] == B
    pred = m((x, sizes), eps=eps)
    assert np.abs(pred - fr.pred).max() < 2e-5 * max(1.0, np.abs(fr.pred).max())
    # the set transformer alone on the reparameterised embeddings (padding rows arbitrary)
    c = VO.forward(cfg, p, x, eps, sizes, keep=True).cache
    E = cfg.bottleneck_dimension
    u = (c["mu"] + np.exp(c["lv"] / 2) * eps.reshape(-1, E)).reshape(B, cfg.number_particles, E).astype(np.float32)
    u[VO.mask_of(sizes, cfg.number_particles) == 0] = np.nan
    assert np.abs(m.set_transformer(u, set_sizes=sizes) - fr.pred).max() < 2e-5 * max(1.0, np.abs(fr.pred).max())


def test_matches_the_fixed_size_model_at_each_size():
    cfg = small(64)
    for l in (1, 13, 64):                                             # a uniform batch of size l = the fixed model at L = l
        p, x, y, eps, _ = varlen_set_case(cfg, [l] * 6, 2)
        fixed = set_transformer_model(small(l))
        var = set_transformer_model(cfg, variable=True)
        for mm in (fixed, var):
            mm.set_flat_weights(p)
            mm.beta.assign(0.05)
        gf, sf = fixed.compute_gradients(x[:, :l], y, eps=eps[:, :l])
        gv, sv = var.compute_gradients((x, np.full(6, l, np.int32)), y, eps=eps)
        assert rel_err(gv.cpu().numpy(), gf.cpu().numpy()) < 1e-5, l
        np.testing.assert_allclose(sv.cpu().numpy(), sf.cpu().numpy(), rtol=1e-5)
    sizes = np.array([1, 13, 64, 40, 2], np.int32)                    # per-set predictions of a mixed batch
    p, x, y, eps, _ = varlen_set_case(cfg, sizes, 3)
    var = set_transformer_model(cfg, variable=True)
    var.set_flat_weights(p)
    pv = var((x, sizes), eps=eps)
    for s, l in enumerate(sizes):
        fixed = set_transformer_model(small(int(l)))
        fixed.set_flat_weights(p)
        pf = fixed(x[s:s + 1, :l], eps=eps[s:s + 1, :l])
        assert np.abs(pv[s] - pf[0]).max() < 1e-5 * max(1.0, np.abs(pf).max()), l


def test_padding_content_is_ignored_bit_for_bit():
    cfg = small(65)
    sizes = np.array([1, 65, 30, 64, 2, 17], np.int32)
    p, x, y, eps, _ = varlen_set_case(cfg, sizes, 4)
    pad = VO.mask_of(sizes, cfg.number_particles) == 0
    xz, xn, en = x.copy(), x.copy(), eps.copy()
    xz[pad], xn[pad], en[pad] = 0.0, np.nan, np.inf
    m = set_transformer_model(cfg, variable=True)
    m.set_flat_weights(p)
    m.beta.assign(0.1)
    out = []
    for xx, ee in ((xz, eps), (xn, en)):
        g, st = m.compute_gradients((xx, sizes), y, eps=ee)
        out.append((g.cpu().numpy(), st.cpu().numpy(), m((xx, sizes), eps=ee), m.predict((xx, sizes), batch_size=4)))
    for a, b in zip(out[0][:3], out[1][:3]):
        assert np.isfinite(a).all() and np.array_equal(a, b)
    assert np.isfinite(out[1][3]).all()
    # Philox noise too: padding rows draw noise nobody reads
    g1, _ = m.compute_gradients((xz, sizes), y, step=9)
    g2, _ = m.compute_gradients((xn, sizes), y, step=9)
    assert torch.equal(g1, g2)


def test_shards_add_up_to_the_full_batch():
    cfg = small(7)
    sizes = np.array([1, 7, 3, 7, 5, 1, 2, 6, 4, 7, 2, 3], np.int32)
    B = len(sizes)
    m = set_transformer_model(cfg, variable=True)
    p, x, y, eps, _ = varlen_set_case(cfg, sizes, 5)
    m.set_flat_weights(p)
    m.beta.assign(0.1)
    for kw in (lambda a, b: dict(eps=eps[a:b]), lambda a, b: dict(step=3)):
        g, st = m.compute_gradients((x, sizes), y, **kw(0, B))
        g1, s1 = m.compute_gradients((x[:5], sizes[:5]), y[:5], global_batch=B, **kw(0, 5))
        g2, s2 = m.compute_gradients((x[5:], sizes[5:]), y[5:], global_batch=B, sample_offset=5, **kw(5, B))
        assert rel_err((g1 + g2).cpu().numpy(), g.cpu().numpy()) < 1e-5
        np.testing.assert_allclose((s1 + s2).cpu().numpy(), st.cpu().numpy(), rtol=1e-5)


def test_seeded_runs_and_graph_replay_with_changing_sizes_are_bit_identical():
    cfg, B = small(70), 16
    p, x, y, _, _ = varlen_set_case(cfg, [1] * B, 6)
    a = set_transformer_model(cfg, variable=True)
    a.set_flat_weights(p)
    s0 = _sizes(1, 70, B, 7)
    g1, t1 = a.compute_gradients((x, s0), y, step=5)
    g2, t2 = a.compute_gradients((x, s0), y, step=5)
    assert torch.equal(g1, g2) and torch.equal(t1, t2)
    size_steps = [_sizes(1, 70, B, 10 + k) for k in range(6)]
    runs = []
    for graph in (False, True):
        m = set_transformer_model(cfg, variable=True)
        m.use_cuda_graph = graph
        m.set_flat_weights(p)
        m.beta.assign(0.05)
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        stats = [m.train_on_batch((xd, torch.from_numpy(s).cuda()), yd)["loss"] for s in size_steps]
        assert (len(m._graphs) > 0) == graph
        runs.append((m.get_flat_weights(), stats))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert runs[0][1] == runs[1][1]


def test_fit_on_a_ragged_list_follows_the_oracle_history():
    import dib_b200
    cfg, B, n, nv = small(7), 8, 28, 10
    m = set_transformer_model(cfg, variable=True, lr=2e-3, metrics=["accuracy"])
    m.noise_seed = 77
    sizes = _sizes(1, 7, n + nv, 8)
    sizes[:2] = (1, 7)
    p, x, y, _, _ = varlen_set_case(cfg, sizes, 9)
    sets = [x[i, :sizes[i]] for i in range(n + nv)]                   # the notebook's list before np.stack
    m.set_flat_weights(p)
    cb = dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)
    hist = m.fit(sets[:n], y[:n], batch_size=B, epochs=3, callbacks=[cb], validation_data=(sets[n:], y[n:]), verbose=0).history
    perms = {e: m.epoch_permutation(e, n).cpu().numpy() for e in range(3)}
    L, E = cfg.number_particles, cfg.bottleneck_dimension

    def eps_fn(step, set_ids):
        rows = (np.asarray(set_ids)[:, None] * L + np.arange(L)[None, :]).ravel()
        return philox.normal_noise(77, step, rows, 1, E, dtype=np.float64).reshape(len(set_ids), L, E)
    xp, sp = dib_b200.pad_sets(sets, L)
    _, h_ref = VO.fit(cfg, p, xp[:n].astype(np.float64), y[:n].astype(np.float64), sp[:n], epochs=3, batch_size=B, lr=2e-3,
                      eps_fn=eps_fn, perm_fn=lambda e, N: perms[e], beta_fn=lambda e: O.beta_schedule(e, 1e-3, 1e-1, 1, 2),
                      validation_data=(xp[n:].astype(np.float64), y[n:].astype(np.float64), sp[n:]))
    assert set(hist) == set(h_ref)
    for k in h_ref:
        np.testing.assert_allclose(hist[k], h_ref[k], rtol=2e-3, atol=1e-6, err_msg=k)
    # evaluate / predict on the list, and the particle encoder on the list and on the padded pair
    ev = m.evaluate(sets[n:], y[n:], batch_size=4)
    assert np.isfinite(ev["loss"])
    assert m.predict(sets[n:], batch_size=3).shape == (nv, 1)
    ml = m.particle_encoder(sets[n:])
    mp = m.particle_encoder((xp[n:], sp[n:]))
    for i, a in enumerate(ml):
        assert a.shape == (sp[n + i], 2 * E)
        np.testing.assert_array_equal(a, mp[i, :sp[n + i]])
        assert (mp[i, sp[n + i]:] == 0).all()


def test_tf32_against_fp32():
    cfg = NOTEBOOK100
    sizes = _sizes(20, 100, 32, 11)
    p, x, y, eps, _ = varlen_set_case(cfg, sizes, 12)
    out = {}
    for prec in ("fp32", "tf32"):
        m = set_transformer_model(cfg, variable=True, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(0.02)
        g, st = m.compute_gradients((x, sizes), y, eps=eps)
        out[prec] = (g.cpu().numpy(), st.cpu().numpy(), m((x, sizes), eps=eps))
    eg, ep = rel_err(out["tf32"][0], out["fp32"][0]), np.abs(out["tf32"][2] - out["fp32"][2]).max()
    print(f"variable sizes, tf32 vs fp32: gradient max-norm rel {eg:.3e}, prediction abs {ep:.3e}")
    assert eg < 3e-2 and ep < 1e-2
    assert abs(out["tf32"][1][0] - out["fp32"][1][0]) < 5e-3 * abs(out["fp32"][1][0])


def test_dib_create_limits_and_unbound_sizes():
    from dib_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    for L in (1, 65, 256):
        cfg, _ = _config(set_size=L, variable_set_sizes=1)
        assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) == 0, lib.dib_last_error()
        lib.dib_destroy(h)
    cfg, _ = _config(set_size=257, variable_set_sizes=1)
    assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
    assert "[1, 256]" in lib.dib_last_error().decode()
    cfg, _ = _config(set_size=65)
    assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) != 0 and "set_size" in lib.dib_last_error().decode()
    # a variable-size handle without bound sizes refuses to run; a fixed-size handle refuses sizes
    m = set_transformer_model(small(7), variable=True)
    m._ensure_handle(4)
    x = torch.zeros(4, 7 * 3, device="cuda")
    stats = torch.empty(4, device="cuda")
    assert lib.dib_forward(m._handle, _lib.ptr(m._params), _lib.ptr(x), None, 4, _lib.ptr(m.beta._dev), None, 0, 0, 0, None, None,
                           _lib.ptr(stats), _lib.ptr(m._workspace), None) != 0
    assert "dib_set_set_sizes_device" in lib.dib_last_error().decode()
    f = set_transformer_model(small(7))
    f._ensure_handle(4)
    sz = torch.ones(4, dtype=torch.int32, device="cuda")
    assert lib.dib_set_set_sizes_device(f._handle, _lib.ptr(sz)) != 0
