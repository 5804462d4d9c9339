"""GPU (H100): per-sample weights of the compiled loss (fit / evaluate / train_on_batch sample_weight=, class_weight=) on
every loss kernel -- dib_loss_kernel (fp32 / tf32 / the set transformer's head), dib_int16_head_kernel, dib_int16_head1_kernel
and the fused tail dib_int16_fwd2_kernel -- against the float64 oracles with weights, and all-ones weights against the
unweighted launches bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import fused16_oracle as Q
from tests import sample_weight_oracle as SW
from tests.test_gpu_parity import build_model, make_labels, rel_err
from tests.test_gpu_fused16_vs_rounding_oracle import TOL, _c, _check, _data, _expect_route, _model, _params

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _weights(n, seed, hi=50.0):
    """Weights in [0, hi] with zeros and a few exact integers."""
    rng = np.random.default_rng(seed + 77)
    w = rng.uniform(0.0, hi, n).astype(np.float32)
    w[rng.choice(n, max(1, n // 10), replace=False)] = 0.0
    w[:3] = [0.0, 1.0, hi]
    return w


def _grads(m, x, y, eps, w=None):
    g, st = m.compute_gradients(x, y, eps=eps, sample_weight=w)
    return g.cpu().numpy(), st.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# fp32 against the float64 oracle (bounds of test_gpu_parity.py)
# ---------------------------------------------------------------------------------------------------------------------
FP32_CASES = {
    "bce_logits": (O.LOSS_BCE_LOGITS, 1, None), "bce_probs": (O.LOSS_BCE_PROBS, 1, "sigmoid"),
    "sce3": (O.LOSS_SPARSE_CE_LOGITS, 3, None), "sce8": (O.LOSS_SPARSE_CE_LOGITS, 8, None),
    "mse1": (O.LOSS_MSE, 1, None), "mse6": (O.LOSS_MSE, 6, None),
}
LOSS_NAME = {O.LOSS_BCE_LOGITS: "bce_logits", O.LOSS_BCE_PROBS: "bce_probs", O.LOSS_SPARSE_CE_LOGITS: "sparse_ce_logits",
             O.LOSS_MSE: "mse"}


@pytest.mark.parametrize("n", [127, 4173])
@pytest.mark.parametrize("case", list(FP32_CASES))
def test_fp32_weighted_step_matches_oracle(case, n):
    loss, out, out_act = FP32_CASES[case]
    cfg = O.DIBConfig([1, 2, 1, 3], [32, 32], [64, 32], out, feature_embedding_dimension=8, activation_fn="tanh",
                      output_activation_fn=out_act)
    rng = np.random.default_rng(n)
    p = O.glorot_uniform_params(cfg, rng)
    x = rng.standard_normal((n, 7)).astype(np.float32)
    eps = rng.standard_normal((n, 4, 8)).astype(np.float32)
    y = make_labels(rng, loss if loss != O.LOSS_BCE_PROBS else O.LOSS_BCE_LOGITS, n, out)
    w = _weights(n, n)
    m = build_model(cfg, loss=LOSS_NAME[loss])
    m.set_flat_weights(p)
    m.beta.assign(0.05)
    g, st = _grads(m, x, y, eps, w)
    g_ref, fr = SW.train_grads(cfg, p, x, y, eps, 0.05, loss, w)
    assert rel_err(g, g_ref) < 5e-5
    off = 0
    for s in cfg.param_shapes():
        k = int(np.prod(s))
        assert rel_err(g[off:off + k], g_ref[off:off + k]) < 2e-4, (off, s)
        off += k
    F = cfg.number_features
    np.testing.assert_allclose(st[:F] / n, fr.kl_per_feature, rtol=2e-5)
    np.testing.assert_allclose(st[F] / n, fr.task_loss, rtol=2e-5)          # sum_i w_i l_i
    np.testing.assert_allclose(st[F + 1], fr.acc_sum, rtol=1e-6)            # accuracy: unweighted
    key = (1 << 29) | (m._inference_calls + 1)                                 # evaluate's noise key
    logs = m.evaluate(x, y, batch_size=n, sample_weight=w)
    ev = SW.forward(cfg, m.get_flat_weights(), x, philox.normal_noise(m.noise_seed, 2 ** 31 + key, np.arange(n), F, 8,
                                                                       dtype=np.float64), 0.05, y, loss, w)
    np.testing.assert_allclose(logs["loss"], ev.loss, rtol=2e-5)


# ---------------------------------------------------------------------------------------------------------------------
# all-ones weights: the unweighted bits, on every loss kernel
# ---------------------------------------------------------------------------------------------------------------------
ONES = {
    # name: (cfg kwargs, loss, precision, debug mask, route)
    "c0_fp16_fused_tail": (dict(F=16), "bce_logits", "fp16", 0, "dgrad"),
    "c0_bf16_fused_tail": (dict(F=16), "bce_logits", "bf16", 0, "dgrad"),
    "c0_fp16_tail_fwd2": (dict(F=16), "mse", "fp16", 16, "fwd2"),
    "head1_fp16": (dict(F=16, integ=(128, 256)), "bce_logits", "fp16", 0, None),
    "head1_bf16_probs": (dict(F=16, integ=(128, 256), probs=True), "bce_probs", "bf16", 0, None),
    "head6_fp16_mse": (dict(F=16, out=6), "mse", "fp16", 0, None),
    "head3_bf16_sce": (dict(F=16, out=3), "sparse_ce_logits", "bf16", 0, None),
}


@pytest.mark.parametrize("name", list(ONES))
def test_all_ones_weights_are_bit_identical_16bit(name):
    kw, loss, prec, mask, tail = ONES[name]
    cfg = _c(**kw)
    n = 128 * 9 + 5
    lid = {v: k for k, v in LOSS_NAME.items()}[loss]
    x, y, eps = _data(cfg, lid, n, 2)
    m = _model(cfg, prec, loss, mask)
    _expect_route(m, prec, n, tail)
    m.set_flat_weights(_params(cfg, 2))
    g0, s0 = _grads(m, x, y, eps)
    g1, s1 = _grads(m, x, y, eps, np.ones(n, np.float32))
    assert np.array_equal(g0, g1) and np.array_equal(s0, s1)
    e0, e1 = m.evaluate(x, y, batch_size=n), None
    m._inference_calls -= 1                                                 # the same noise draw again
    e1 = m.evaluate(x, y, batch_size=n, sample_weight=torch.ones(n, device=m.device))
    assert e0 == e1


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
def test_all_ones_weights_are_bit_identical_fp32_tf32(prec):
    cfg = O.DIBConfig([1] * 6, [64, 64], [128, 64], 3, feature_embedding_dimension=16)
    n = 1000
    rng = np.random.default_rng(3)
    x = rng.standard_normal((n, 6)).astype(np.float32)
    eps = rng.standard_normal((n, 6, 16)).astype(np.float32)
    y = rng.integers(0, 3, n).astype(np.float32)
    m = build_model(cfg, precision=prec, loss="sparse_ce_logits")
    m.set_flat_weights(O.glorot_uniform_params(cfg, rng))
    g0, s0 = _grads(m, x, y, eps)
    g1, s1 = _grads(m, x, y, eps, np.ones(n))
    assert np.array_equal(g0, g1) and np.array_equal(s0, s1)


def _set_transformer(varlen, prec="fp32"):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(2, [32], bottleneck_dimension=8, number_particles=12, key_dim=8, number_heads=2,
                                     number_attention_blocks=1, final_processing_arch=[16], precision=prec, seed=1,
                                     variable_set_sizes=varlen)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=["accuracy"])
    return m


@pytest.mark.parametrize("varlen", [False, True])
def test_set_transformer_all_ones_bit_identical_and_weights_act_per_set(varlen):
    rng = np.random.default_rng(5)
    n = 70
    xs = rng.standard_normal((n, 12, 2)).astype(np.float32)
    y = rng.integers(0, 2, (n, 1)).astype(np.float32)
    sizes = rng.integers(1, 13, n).astype(np.int32)
    x = (xs, sizes) if varlen else xs
    m = _set_transformer(varlen)
    g0, s0 = _grads(m, x, y, None)                     # Philox noise keyed by the optimizer step: the same in every call here
    g1, s1 = _grads(m, x, y, None, np.ones(n))
    assert np.array_equal(g0, g1) and np.array_equal(s0, s1)
    # zero weights: no task term, the KL and the accuracy untouched; one weight per set
    _, sz = _grads(m, x, y, None, np.zeros(n))
    assert sz[1] == 0.0 and sz[0] == s0[0] and sz[2] == s0[2]
    # the task-loss statistic is additive over sets: sum_i w_i l_i from the one-hot weights
    w = rng.integers(0, 4, n).astype(np.float32)
    _, sw = _grads(m, x, y, None, w)
    per = np.array([_grads(m, x, y, None, np.eye(n, dtype=np.float32)[i])[1][1] for i in range(n)], np.float64)
    np.testing.assert_allclose(sw[1], (w * per).sum(), rtol=2e-5)
    with pytest.raises(ValueError):
        _grads(m, x, y, None, np.ones(n * 12))                                  # one weight per set, not per particle


# ---------------------------------------------------------------------------------------------------------------------
# fp16 / bf16 against the weighted rounding-aware oracle (bounds of test_gpu_fused16_vs_rounding_oracle.py)
# ---------------------------------------------------------------------------------------------------------------------
SHAPES16 = {
    "F16": (dict(F=16), "bce_logits", 0, "dgrad"),
    "head1": (dict(F=16, integ=(128, 256)), "bce_logits", 0, None),
    "sce3": (dict(F=16, out=3), "sparse_ce_logits", 0, None),
    "mse3": (dict(F=16, out=3), "mse", 0, None),
    "mask16": (dict(F=16), "bce_logits", 16, "fwd2"),
    "probs": (dict(F=12, probs=True), "bce_probs", 0, "dgrad"),
}


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", list(SHAPES16))
def test_16bit_weighted_step_matches_rounding_oracle(shape, prec):
    kw, loss, mask, tail = SHAPES16[shape]
    cfg = _c(**kw)
    lid = {v: k for k, v in LOSS_NAME.items()}[loss]
    n = 128 * 32 + 77
    p = _params(cfg, 3)
    x, y, eps = _data(cfg, lid, n, 3)
    w = _weights(n, 3)
    m = _model(cfg, prec, loss, mask)
    _expect_route(m, prec, n, tail)
    m.set_flat_weights(p)
    m.beta.assign(1e-3)
    g, st = _grads(m, x, y, eps, w)
    assert np.isfinite(g).all() and np.isfinite(st).all()
    g_ref, fr = SW.fused16_train_grads(cfg, p, x, y, eps, 1e-3, lid, w, fmt=prec)
    pv = Q.per_variable_errors(cfg, g.astype(np.float64), g_ref)
    _check(f"weighted grad/var {shape} {prec}", pv.max(), TOL[("grad", prec)])
    F = cfg.number_features
    _check(f"weighted loss sum {shape} {prec}", abs(st[F] - fr.cache["loss_sum"]) / abs(fr.cache["loss_sum"]), TOL[("stats", prec)])


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_zero_weight_step(prec):
    cfg = _c(F=16)
    n = 128 * 9 + 5
    x, y, eps = _data(cfg, O.LOSS_BCE_LOGITS, n, 4)
    m = _model(cfg, prec, "bce_logits")
    _expect_route(m, prec, n, "dgrad")
    m.set_flat_weights(_params(cfg, 4))
    m.beta.assign(0.3)
    g, st = _grads(m, x, y, eps, np.zeros(n, np.float32))
    F = cfg.number_features
    assert st[F] == 0.0
    assert not np.any(g[m._p_enc:])                                            # integration network: exactly 0
    g_kl, _ = m.encoder_gradients(x, np.zeros((n, 16 * 32), np.float32), global_batch=n, eps=eps)
    g_kl = g_kl.cpu().numpy()
    g_ref, _ = SW.fused16_train_grads(cfg, _params(cfg, 4), x, y, eps, 0.3, O.LOSS_BCE_LOGITS, np.zeros(n), fmt=prec)
    err = Q.per_variable_errors(cfg, g.astype(np.float64), g_kl.astype(np.float64))[:-6].max()
    print(f"[sample-weights] zero-weight encoder gradient vs the beta*KL-only gradient {prec}: {err:.3e}")
    assert err < 1e-6
    _check(f"zero-weight grad/var vs oracle {prec}", Q.per_variable_errors(cfg, g.astype(np.float64), g_ref)[:-6].max(),
           TOL[("grad", prec)])


def test_fp16_large_weights_stay_in_range():
    """Weights up to 1e3: the S-scaled 16-bit gradient carries w * (d loss / d z); fp16 against fp32 on the same step."""
    from tests.test_gpu_benched_mode import _c0, _c0_batch
    cfg = _c0()
    B = 4096
    x, y = _c0_batch(B, 7)
    rng = np.random.default_rng(7)
    eps = rng.standard_normal((B, 16, 32)).astype(np.float32)
    w = rng.uniform(0, 1e3, B).astype(np.float32)
    w[:4] = [0.0, 1e3, 1e3, 1e3]
    p = O.glorot_uniform_params(cfg, rng)
    res = {}
    for prec in ("fp32", "fp16"):
        m = build_model(cfg, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(0.01)
        res[prec] = _grads(m, x, y, eps, w)
    g32, g16 = res["fp32"][0], res["fp16"][0]
    assert np.isfinite(g16).all()
    e = rel_err(g16, g32)
    pv = Q.per_variable_errors(cfg, g16.astype(np.float64), g32.astype(np.float64))
    print(f"[sample-weights] fp16 vs fp32, weights up to 1e3: gradient max-norm {e:.3e}, worst variable {pv.max():.3e}")
    assert e < 5e-3                                          # test_fp16_mode_range_edges' fp16-vs-fp32 bounds
    np.testing.assert_allclose(res["fp16"][1], res["fp32"][1], rtol=5e-3)


# ---------------------------------------------------------------------------------------------------------------------
# fit, graph replay, data parallelism
# ---------------------------------------------------------------------------------------------------------------------
def _fit_setup(prec, loss="bce_logits"):
    from tests.test_gpu_benched_mode import _fit_case
    x, y, cfg = _fit_case()
    m = build_model(cfg, precision=prec, lr=1e-3, seed=4)
    m.noise_seed = 99
    return m, x, y, cfg


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_fit_class_weight_equals_sample_weight_and_matches_oracle(prec):
    import dib_b200
    cw = {0: 1.0, 1: 20.0}
    m, x, y, cfg = _fit_setup(prec)
    p0 = m.get_flat_weights().copy()
    rng = np.random.default_rng(1)
    sw = rng.uniform(0, 2, len(x)).astype(np.float32)
    wv = rng.uniform(0, 3, 256).astype(np.float32)
    kw = dict(epochs=3, batch_size=128, verbose=False, validation_data=(x[:256], y[:256], wv))
    h_cw = m.fit(x, y, class_weight=cw, sample_weight=sw, callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)],
                 **kw).history
    p_cw = m.get_flat_weights().copy()
    m2, *_ = _fit_setup(prec)
    w_eq = dib_b200.models.class_weight_rows(y, cw, sw)
    h_sw = m2.fit(x, y, sample_weight=torch.from_numpy(w_eq).cuda(),
                  callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)], **kw).history
    assert h_cw == h_sw and np.array_equal(p_cw, m2.get_flat_weights())          # bit for bit
    perms = {e: m.epoch_permutation(e, len(x)).cpu().numpy() for e in range(3)}
    E, F = cfg.feature_embedding_dimension, cfg.number_features
    eps_fn = lambda step, ids: philox.normal_noise(99, step, ids, F, E, dtype=np.float64)
    _, h_ref = SW.fit(cfg, p0, x.astype(np.float64), y.astype(np.float64), loss=O.LOSS_BCE_LOGITS, epochs=3, batch_size=128,
                     lr=1e-3, eps_fn=eps_fn, perm_fn=lambda e, n: perms[e], beta_fn=lambda e: O.beta_schedule(e, 1e-3, 1e-1, 1, 2),
                     validation_data=(x[:256].astype(np.float64), y[:256].astype(np.float64), wv), sample_weight=w_eq)
    tol = 2e-3 if prec == "fp32" else 3e-2
    assert set(h_cw) == set(h_ref)
    for k in h_ref:
        a, b = np.asarray(h_cw[k], np.float64), np.asarray(h_ref[k], np.float64)
        if "accuracy" in k:
            np.testing.assert_allclose(a, b, atol=3e-2 if prec == "fp16" else 1e-2, err_msg=k)
        else:
            np.testing.assert_allclose(a, b, rtol=tol, atol=1e-4, err_msg=k)
    # class_weight does not touch validation; the validation weights do
    m3, *_ = _fit_setup(prec)
    h_nv = m3.fit(x, y, class_weight=cw, sample_weight=sw, epochs=1, batch_size=128, verbose=False,
                  validation_data=(x[:256], y[:256])).history
    m4, *_ = _fit_setup(prec)
    h_nw = m4.fit(x, y, epochs=1, batch_size=128, verbose=False, validation_data=(x[:256], y[:256])).history
    assert h_nv["loss"][0] != h_nw["loss"][0]
    _, h_v = SW.fit(cfg, p0, x.astype(np.float64), y.astype(np.float64), loss=O.LOSS_BCE_LOGITS, epochs=1, batch_size=128,
                   lr=1e-3, eps_fn=eps_fn, perm_fn=lambda e, n: perms[e],
                   validation_data=(x[:256].astype(np.float64), y[:256].astype(np.float64)), sample_weight=w_eq)
    np.testing.assert_allclose(h_nv["val_loss"], h_v["val_loss"], rtol=tol, atol=1e-4)


def test_graph_replay_with_changing_weights_equals_eager():
    from tests.test_gpu_benched_mode import _c0, _c0_batch
    cfg = _c0()
    x, y = _c0_batch(512, 3)
    rng = np.random.default_rng(3)
    ws = [rng.uniform(0, 5, 512).astype(np.float32) for _ in range(7)]
    out = {}
    for graphs in (True, False):
        m = build_model(cfg, precision="fp16", seed=2)
        m.use_cuda_graph = graphs
        res = [m.train_on_batch(x, y, sample_weight=w) for w in ws]
        res.append(m.train_on_batch(x, y))                                  # an unweighted step after weighted ones
        res += [m.train_on_batch(x, y, sample_weight=w, sync=False).get() for w in ws[:3]]
        out[graphs] = (res, m.get_flat_weights())
        if graphs:
            assert any(k[-1] for k in m._graphs), list(m._graphs)           # a weighted graph was captured and replayed
    assert out[True][0] == out[False][0] and np.array_equal(out[True][1], out[False][1])


def test_train_on_batch_refuses_bad_weights_before_device_work():
    import dib_b200
    from tests.test_gpu_benched_mode import _c0, _c0_batch
    x, y = _c0_batch(64, 1)
    m = build_model(_c0())
    p0 = m.get_flat_weights().copy()
    for bad in (np.ones(63), -np.ones(64), np.full(64, np.nan)):
        with pytest.raises(ValueError):
            m.train_on_batch(x, y, sample_weight=bad)
    with pytest.raises(ValueError):
        m.train_on_batch(x, y, class_weight={0: 1.0})                       # label 1 has no class
    with pytest.raises(ValueError):
        m.fit(x, y, class_weight={1: 1.0, 2: 1.0}, verbose=False)
    assert np.array_equal(p0, m.get_flat_weights()) and m._train_step_count == 0
    mse = build_model(O.DIBConfig([1] * 4, [32], [32], 2), loss="mse")
    with pytest.raises(ValueError):
        mse.fit(np.zeros((8, 4), np.float32), np.zeros((8, 2), np.float32), class_weight={0: 1.0, 1: 2.0}, verbose=False)
    ext = build_model(O.DIBConfig([1] * 4, [32], [32], 1), loss="external")
    with pytest.raises(ValueError):
        ext.compute_gradients(np.zeros((8, 4), np.float32), np.zeros((8, 1), np.float32), sample_weight=np.ones(8))
    import ctypes
    from dib_b200 import _lib
    ext._ensure_handle(8)
    assert _lib.load().dib_set_sample_weights_device(ext._handle, ctypes.c_void_p(16)) != 0


_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["DIB_ROOT"])
import dib_b200
from tests.test_gpu_benched_mode import _fit_case
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(0)
if world > 1:
    dist.init_process_group("gloo")
x, y, cfg = _fit_case()
m = dib_b200.DistributedIBNet(cfg.feature_dimensionalities, cfg.feature_encoder_architecture,
                              cfg.integration_network_architecture, 1, precision=os.environ["DIB_PREC"], seed=4)
m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=["accuracy"])
m.noise_seed = 99
rng = np.random.default_rng(0)
sw, wv = rng.uniform(0, 3, len(x)).astype(np.float32), rng.uniform(0, 3, 256).astype(np.float32)
h = m.fit(x, y, epochs=3, batch_size=128, verbose=False, class_weight={0: 1.0, 1: 5.0}, sample_weight=sw,
          validation_data=(x[:256], y[:256], wv)).history
if rank == 0:
    np.savez(os.environ["DIB_OUT"], params=m.get_flat_weights(), graphs=len(m._graphs), **{k: np.asarray(v) for k, v in h.items()})
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_two_process_gloo_weighted_fit_equals_one_process_fit(tmp_path, prec):
    from tests.test_gpu_infonce_data_parallel import _compare_fits, _free_port
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    res = {}
    for world in (1, 2):
        out = str(tmp_path / f"w{world}.npz")
        env = dict(os.environ, DIB_ROOT=ROOT, DIB_OUT=out, DIB_PREC=prec, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()),
                   WORLD_SIZE=str(world), PYTHONPATH=ROOT)
        procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), cwd=ROOT)
                 for r in range(world)]
        try:
            codes = [pr.wait(timeout=600) for pr in procs]
        finally:
            for pr in procs:
                if pr.poll() is None:
                    pr.kill()
                    pr.wait()
        assert codes == [0] * world, codes
        res[world] = dict(np.load(out))
    # accuracies count rows: the ~1e-7 regrouping of the two ranks' sums may flip a row next to the 0.5 threshold (one of the
    # 256 validation rows in fp16), so they get the absolute bound of the fit test above; everything else _compare_fits' bounds
    acc = [k for k in res[1] if "accuracy" in k]
    for k in acc:
        np.testing.assert_allclose(res[2][k], res[1][k], atol=3e-2 if prec == "fp16" else 1e-2, err_msg=k)
    _compare_fits(*({k: v for k, v in r.items() if k not in acc} for r in (res[1], res[2])), prec)


@pytest.mark.parametrize("varlen", [False, True])
def test_set_transformer_weighted_step_matches_oracle(varlen):
    """Per-set weights against the set-transformer oracles, at the bounds of test_gpu_set_transformer*.py."""
    if varlen:
        from tests.test_gpu_set_transformer_variable_sizes import case, make_model, small
        cfg = small(7)
        p, x, y, eps, sizes = case(cfg, np.array([1, 7, 3, 7, 5, 1, 2, 6, 4], np.int32), 1)
        xin = (x, sizes)
    else:
        from tests.test_gpu_set_transformer import case, make_model, small
        cfg = small(7)
        p, x, y, eps = case(cfg, 9, 1)
        xin = x
    B = x.shape[0]
    w = _weights(B, 9, hi=10.0)
    m = make_model(cfg)
    m.set_flat_weights(p)
    m.beta.assign(0.02)
    g, st = _grads(m, xin, y, eps, w)
    if varlen:
        g_ref, fr = SW.set_transformer_train_grads(cfg, p, x, y, eps, 0.02, O.LOSS_BCE_LOGITS, w, sizes=sizes)
    else:
        g_ref, fr = SW.set_transformer_train_grads(cfg, p, x, y, eps, 0.02, O.LOSS_BCE_LOGITS, w)
    assert rel_err(g, g_ref) < 5e-5
    scale = np.abs(g_ref).max()
    for i in range(len(m._var_off)):
        off, n = m._var_off[i], max(m._var_rows[i], 1) * m._var_cols[i]
        ref = np.abs(g_ref[off:off + n]).max()
        assert np.abs(g[off:off + n] - g_ref[off:off + n]).max() < 2e-4 * max(ref, 1e-3 * scale), i
    assert abs(st[0] / B - fr.kl) < 2e-5 * max(1.0, fr.kl)
    assert abs(st[1] / B - fr.task_loss) < 2e-5 * max(1.0, fr.task_loss)
