"""GPU (H100): training with losses.InfoNCE (train.py:180-289) -- the output encoder and the streaming InfoNCE kernels --
against the float64 oracle (tests/infonce_oracle.py), the existing materialised InfoNCE head, a float64 evaluation at a
batch above that head's limit, and itself (determinism, graph replay)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import infonce_oracle as IO

pytestmark = pytest.mark.gpu

# the double-pendulum shape of train.py:116-126 / BASELINE config 3: features [2, 1, 2, 1], out = infonce dim 64,
# output encoder 6 -> PE 30 -> [128, 128] -> 64
CFG = O.DIBConfig([2, 1, 2, 1], [128, 128], [256, 256], 64)
YD, YARCH = 6, [128, 128]


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def make_model(similarity="l2", temperature=1.0, precision="fp32", seed=0, lr=1e-3, **kw):
    import dib_b200
    m = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                                  CFG.integration_network_architecture, CFG.output_dimensionality, output_activation_fn=None,
                                  precision=precision, seed=seed, **kw)
    m.compile(optimizer=dib_b200.Adam(lr), loss=dib_b200.losses.InfoNCE(YD, YARCH, similarity=similarity,
                                                                        temperature=temperature))
    return m


def data(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 6)).astype(np.float32)
    y = np.stack([np.sin(x[:, 0]) * x[:, 1], x[:, 2] * x[:, 3], np.cos(x[:, 4]), x[:, 5] ** 2 - 1, np.tanh(x[:, 0] + x[:, 4]),
                  x[:, 1] * x[:, 5]], -1).astype(np.float32)
    eps = rng.standard_normal((n, 4, 32)).astype(np.float32)
    return x, y, eps


def params(seed):
    rng = np.random.default_rng(seed)
    return IO.glorot(IO.infonce_param_shapes(CFG, YD, YARCH), rng).astype(np.float32)


def temperature_of(similarity):
    return 0.1 if similarity == "cosine" else 1.0


@pytest.mark.parametrize("n", [512, 4160])
@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_fp32_step_matches_float64_oracle(similarity, n):
    T = temperature_of(similarity)
    m = make_model(similarity, T)
    p = params(1)
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    x, y, eps = data(n, 2)
    g, st = m.compute_gradients(x, y, eps=eps)
    g, st = g.cpu().numpy(), st.cpu().numpy()
    g_ref, loss_ref, kl_ref = IO.infonce_train_grads(CFG, p, x, y, eps, 0.01, y_dimensionality=YD, y_encoder_architecture=YARCH,
                                                     similarity=similarity, temperature=T)
    assert rel_err(g, g_ref) < 5e-5, similarity
    for i, v in enumerate(m.trainable_variables):        # model variables, then the output encoder's (train.py:198)
        off = m._var_off[i]
        sl = slice(off, off + v.numel())
        assert rel_err(g[sl], g_ref[sl]) < 2e-4, (similarity, i)
    F = CFG.number_features
    assert abs(st[F] / n - loss_ref) < 2e-5 * max(1.0, abs(loss_ref))
    np.testing.assert_allclose(st[:F] / n, kl_ref, rtol=2e-5, atol=1e-7)
    assert st[F + 1] == 0 and st[F + 2] == n
    _, layers = IO.split_params(CFG, p, YD, YARCH)
    e2 = m.output_encoder(y)
    assert rel_err(e2, IO.output_encoder_forward(CFG, layers, y)) < 2e-5


@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_step_agrees_with_the_materialised_head_recipe(similarity):
    """The compiled step's model-side gradient equals the recipe it replaces: model(x) and output_encoder(y), the
    materialised head (utils.infonce_loss_and_grads), then compute_gradients of a loss='external' twin."""
    import dib_b200
    from dib_b200 import utils
    T = temperature_of(similarity)
    n = 512
    m = make_model(similarity, T)
    p = params(3)
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    x, y, eps = data(n, 4)
    g, st = m.compute_gradients(x, y, eps=eps)
    e1 = m(torch.from_numpy(x).cuda(), eps=eps)
    e2 = m.output_encoder(torch.from_numpy(y).cuda())
    loss, d_e1, _ = utils.infonce_loss_and_grads(e1, e2, similarity, T)
    twin = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                                     CFG.integration_network_architecture, CFG.output_dimensionality)
    twin.compile(optimizer=dib_b200.Adam(1e-3), loss="external")
    px = CFG.param_count()
    assert twin.count_params() == px
    twin.set_flat_weights(p[:px])
    twin.beta.assign(0.01)
    g_ext, _ = twin.compute_gradients(x, d_e1, eps=eps)
    assert rel_err(g.cpu().numpy()[:px], g_ext.cpu().numpy()) < 1e-5, similarity
    F = CFG.number_features
    assert abs(st[F].item() / n - loss.item()) <= 1e-6 * abs(loss.item())


def test_large_batch_beyond_the_materialised_head():
    n = 40000
    m = make_model("l2", 1.0)
    p = params(5)
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    x, y, eps = data(n, 6)
    _, st = m.compute_gradients(x, y, eps=eps)
    e1 = m(torch.from_numpy(x).cuda(), eps=eps).double()
    e2 = m.output_encoder(torch.from_numpy(y).cuda()).double()
    # float64 InfoNCE on the same embeddings, 4096 rows of the similarity matrix at a time
    col = torch.full((n,), -float("inf"), dtype=torch.float64, device=e1.device)
    tot = 0.0
    b2 = (e2 * e2).sum(-1)
    for i0 in range(0, n, 4096):
        a = e1[i0:i0 + 4096]
        S = -torch.sqrt(torch.clamp((a * a).sum(-1)[:, None] + b2[None, :] - 2.0 * a @ e2.T, min=0.0) + 1e-9)
        tot += (torch.logsumexp(S, 1) - 2.0 * S.diagonal(offset=i0)).sum().item()
        col = torch.logaddexp(col, torch.logsumexp(S, 0))
    ref = (tot + col.sum().item()) / n
    F = CFG.number_features
    assert abs(st[F].item() / n - ref) < 1e-5 * abs(ref), (st[F].item() / n, ref)
    lib = m._lib
    m._release_handle()
    m._ensure_handle(20000)
    w20 = int(lib.dib_workspace_bytes(m._handle))
    m._ensure_handle(40000)
    w40 = int(lib.dib_workspace_bytes(m._handle))
    assert w40 < 2.2 * w20, (w20, w40)


@pytest.mark.parametrize("precision,tol,grad_tol", [("tf32", 5e-3, 3e-2), ("fp16", 5e-3, 3e-2), ("bf16", 4e-2, 4e-2)])
def test_tensor_core_precisions_against_fp32(precision, tol, grad_tol):
    """Embeddings and the loss stay within DESIGN section 2's bounds for the mode.  The gradient bound is wider for tf32 /
    fp16: d e1_i = sum_j w_ij d s_ij / d e1_i with weights that sum to ~0 over j, so the ~7e-4 relative error of the TF32
    embeddings comes out ~25x larger in the gradients (1.7e-2 measured on an H100; the loss moves by ~2e-6)."""
    n = 1024
    p = params(7)
    x, y, eps = data(n, 8)
    out = {}
    for prec in ("fp32", precision):
        m = make_model("l2", 1.0, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(0.01)
        g, st = m.compute_gradients(x, y, eps=eps)
        e1 = m(torch.from_numpy(x).cuda(), eps=eps).cpu().numpy()
        e2 = m.output_encoder(torch.from_numpy(y).cuda()).cpu().numpy()
        out[prec] = (g.cpu().numpy(), st.cpu().numpy(), e1, e2, m.kernel_info(n))
    g32, st32, e1_32, e2_32, info32 = out["fp32"]
    g, st, e1, e2, info = out[precision]
    assert rel_err(e1, e1_32) < tol and rel_err(e2, e2_32) < tol, (rel_err(e1, e1_32), rel_err(e2, e2_32))
    F = CFG.number_features
    assert abs(st[F] - st32[F]) < tol * abs(st32[F])
    np.testing.assert_allclose(st[:F], st32[:F], rtol=tol)
    assert rel_err(g, g32) < grad_tol, (precision, rel_err(g, g32))
    assert "output_encoder=wgmma-tf32" in info and "loss=infonce-stream-fp32" in info, info
    assert "output_encoder=simt-fp32" in info32 and "loss=infonce-stream-fp32" in info32, info32


def test_graph_replay_and_seeded_runs_are_bit_identical():
    x, y, _ = data(2048, 9)
    p = params(11)
    runs = []
    for graphs in (True, False, False):
        m = make_model("l2", 1.0, seed=3)
        m.use_cuda_graph = graphs
        m.set_flat_weights(p)
        m.beta.assign(0.01)
        outs = [m.train_on_batch(x[k * 512:(k + 1) * 512], y[k * 512:(k + 1) * 512])["loss"] for k in range(4)
                for _ in range(2)]
        if graphs:
            assert m._graphs, "the InfoNCE step was not captured"
        runs.append((m.get_flat_weights().copy(), outs))
    for w, o in runs[1:]:
        np.testing.assert_array_equal(w, runs[0][0])
        assert o == runs[0][1]


def test_fit_matches_oracle_and_learns():
    import dib_b200
    n, nv, B = 1100, 300, 256
    x, y, _ = data(n + nv, 12)
    m = make_model("l2", 1.0, seed=4, lr=2e-3)
    m.noise_seed = 99
    p0 = m.get_flat_weights().copy()
    cb = dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 3)
    hist = m.fit(x[:n], y[:n], epochs=4, batch_size=B, callbacks=[cb], verbose=False, validation_data=(x[n:], y[n:])).history
    F = CFG.number_features
    keys = {"loss", "beta", "val_loss", "val_beta"} | {f"{p}KL{i}" for p in ("", "val_") for i in range(F)}
    assert set(hist) == keys
    perms = {e: m.epoch_permutation(e, n).cpu().numpy() for e in range(4)}
    vperms = {e: m.validation_permutation(e, nv).cpu().numpy() for e in range(4)}
    eps_fn = lambda step, ids: philox.normal_noise(99, step, ids, F, 32, dtype=np.float64)
    _, h_ref = IO.fit_infonce(CFG, p0, x[:n].astype(np.float64), y[:n].astype(np.float64), epochs=4, batch_size=B, lr=2e-3,
                              eps_fn=eps_fn, perm_fn=lambda e, N: perms[e], val_perm_fn=lambda e, N: vperms[e],
                              beta_fn=lambda e: O.beta_schedule(e, 1e-3, 1e-1, 1, 3),
                              validation_data=(x[n:].astype(np.float64), y[n:].astype(np.float64)),
                              y_dimensionality=YD, y_encoder_architecture=YARCH)
    assert set(h_ref) == keys
    for k in h_ref:
        np.testing.assert_allclose(hist[k], h_ref[k], rtol=2e-3, atol=1e-6, err_msg=k)

    # a pendulum-like synthetic (y a fixed nonlinear function of x): the InfoNCE term falls
    m = make_model("l2", 1.0, seed=5, lr=1e-3)
    m.beta.assign(1e-3)
    xs, ys, _ = data(8 * 512, 13)
    terms = []
    for step in range(60):
        k = step % 8
        r = m.train_on_batch(xs[k * 512:(k + 1) * 512], ys[k * 512:(k + 1) * 512])
        terms.append(r["loss"] - 1e-3 * sum(r[f"KL{i}"] for i in range(F)))
    assert np.mean(terms[-5:]) < 0.8 * np.mean(terms[:5]), terms


def test_rejections_and_abi_2_configs(monkeypatch):
    import dib_b200
    from dib_b200 import _lib, parallel
    nce = dib_b200.losses.InfoNCE(YD, YARCH)
    m = dib_b200.DistributedIBNet([2, 1], [16], [16], 8, output_activation_fn=None)
    with pytest.raises(ValueError, match="accuracy"):
        m.compile(loss=nce, metrics=["accuracy"])
    with pytest.raises(ValueError, match="losses.InfoNCE"):
        m.compile(loss="infonce")
    ms = dib_b200.DistributedIBNet([2, 1], [16], [16], 8, output_activation_fn="sigmoid")
    with pytest.raises(ValueError, match="output_activation_fn"):
        ms.compile(loss=nce)
    p_model = m.count_params()
    m.compile(loss=nce)
    assert m.count_params() > p_model and m.output_encoder is not None
    x = np.zeros((64, 3), np.float32)
    with pytest.raises(ValueError, match="output encoder"):
        m.fit(x, np.zeros((64, YD + 1), np.float32), batch_size=32, verbose=False)
    with pytest.raises(ValueError, match="full batch"):
        m.fit(x[:16], np.zeros((16, YD), np.float32), batch_size=32, verbose=False)
    m.compile(loss="mse")                                   # back to a compiled loss: the output encoder goes
    assert m.count_params() == p_model and m.output_encoder is None
    monkeypatch.setattr(parallel, "world_and_rank", lambda group=None: (2, 0))
    with pytest.raises(NotImplementedError, match="all-gather"):
        m.compile(loss=nce)
    monkeypatch.undo()

    class DibConfigV2(ctypes.Structure):                    # the ABI-2 struct: every field before the InfoNCE ones
        _fields_ = _lib.DibConfig._fields_[:22]
    assert DibConfigV2._fields_[-1][0] == "dropout_rate"
    lib = _lib.load()
    ref = m._config(1)
    cfg2 = DibConfigV2(**{name: getattr(ref, name) for name, _ in DibConfigV2._fields_})
    cfg2.abi_version = 2
    h = ctypes.c_void_p()
    _lib.check(lib.dib_create(ctypes.cast(ctypes.pointer(cfg2), ctypes.POINTER(_lib.DibConfig)), ctypes.byref(h)))
    try:
        assert lib.dib_param_count(h) == p_model
    finally:
        lib.dib_destroy(h)
