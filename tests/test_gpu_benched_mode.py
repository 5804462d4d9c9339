"""GPU (H100): parity of the mode bench.py reports -- precision='fp16' (fused wgmma kernels: fp16
operands with a 10-bit explicit mantissa, fp32 accumulation, power-of-two loss scale on the gradient operands) -- at
the metric's own batch size, over a training trajectory, at the edge of fp16's range, and across two GPUs.

Tolerances (stated here, asserted below):
  * one step at C0 / B=65 536 vs the exact-fp32 CUDA path (itself pinned to the float64 oracle at 5e-5):
    gradients 5e-3 max-norm overall and 2e-2 per variable, statistics 5e-3 relative;
  * `fit` trajectory (beta annealed, validation every epoch) vs the float64 oracle's fit with the same shuffles and
    noise: every loss / KL{i} / val_ series within 3e-2 relative (+1e-4 absolute), accuracies within 3e-2 absolute --
    ~8x the per-step bound, for 32 chained Adam steps;
  * N-GPU == 1-GPU: identical arithmetic per sample, different fp32 summation grouping, amplified by Adam over 12 steps ->
    2e-4 in the fp32 mode, 5e-3 on the weights / 2e-3 on the history in the fp16 mode.
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests.test_gpu_parity import build_model, rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c0():
    return O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)


def _c0_batch(B, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, 16)).astype(np.float32)
    y = (x[:, 0] * x[:, 1] + np.sin(2 * x[:, 2]) + 0.5 * x[:, 3] > 0).astype(np.float32)[:, None]
    return x, y


def _per_variable(cfg, g, g_ref):
    off, worst = 0, (0.0, None)
    for s in cfg.param_shapes():
        n = int(np.prod(s))
        e = rel_err(g[off:off + n], g_ref[off:off + n])
        if e > worst[0]:
            worst = (e, (off, s))
        off += n
    return worst


@pytest.mark.parametrize("beta", [1e-3, 1.0])
def test_fp16_mode_full_metric_batch_matches_fp32_path(beta):
    """C0 at the metric batch B = 65 536 (loss scale S = 65 536): gradients and statistics of the benched mode against
    the exact-fp32 path on the same weights, inputs and in-kernel Philox noise."""
    cfg = _c0()
    B = 65536
    x, y = _c0_batch(B)
    p = O.glorot_uniform_params(cfg, np.random.default_rng(1))
    p = p + (p == 0) * (0.05 * np.random.default_rng(2).standard_normal(p.size)).astype(np.float32)   # non-zero biases
    out = {}
    for prec in ("fp32", "fp16"):
        m = build_model(cfg, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(beta)
        g, st = m.compute_gradients(x, y, step=3)
        g2, st2 = m.compute_gradients(x, y, step=3)
        assert torch.equal(g, g2) and torch.equal(st, st2)                      # bit-reproducible
        out[prec] = (g.cpu().numpy(), st.cpu().numpy())
        del m
    assert "fused-wgmma-f16" in build_model(cfg, precision="fp16").kernel_info(B)
    g16, g32 = out["fp16"][0], out["fp32"][0]
    assert np.isfinite(g16).all()
    assert rel_err(g16, g32) < 5e-3
    worst = _per_variable(cfg, g16, g32)
    assert worst[0] < 2e-2, worst
    np.testing.assert_allclose(out["fp16"][1], out["fp32"][1], rtol=5e-3)
    # shard additivity in the benched mode (what the data-parallel all-reduce relies on)
    m = build_model(cfg, precision="fp16")
    m.set_flat_weights(p)
    m.beta.assign(beta)
    h = B // 2
    ga, sa = m.compute_gradients(x[:h], y[:h], global_batch=B, sample_offset=0, step=3)
    gb, sb = m.compute_gradients(x[h:], y[h:], global_batch=B, sample_offset=h, step=3)
    assert rel_err((ga + gb).cpu().numpy(), g16) < 2e-4
    np.testing.assert_allclose((sa + sb).cpu().numpy(), out["fp16"][1], rtol=1e-5)


def _fit_case():
    """Boolean circuit (data.py:40; SURVEY 8d C1) on a fused-path-eligible model: 10 features, encoders [128,128],
    E=32, integration [256], 4 epochs x 8 steps, beta annealed 1e-3 -> 1e-1 after one pre-training epoch."""
    x, y = O.boolean_circuit_truth_table()
    cfg = O.DIBConfig([1] * 10, [128, 128], [256], 1)
    return x, y, cfg


def test_fp16_mode_fit_trajectory_matches_oracle():
    import dib_b200
    x, y, cfg = _fit_case()
    m = build_model(cfg, precision="fp16", lr=1e-3, seed=4)
    assert "fused-wgmma-f16" in m.kernel_info(128) and "int16-wgmma-f16" in m.kernel_info(128)
    m.noise_seed = 99
    p0 = m.get_flat_weights().copy()
    E, F = cfg.feature_embedding_dimension, cfg.number_features
    cb = dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 3)
    hist = m.fit(x, y, epochs=4, batch_size=128, shuffle=True, callbacks=[cb], verbose=False,
                 validation_data=(x[:256], y[:256])).history
    perms = {e: m.epoch_permutation(e, 1024).cpu().numpy() for e in range(4)}
    eps_fn = lambda step, ids: philox.normal_noise(99, step, ids, F, E, dtype=np.float64)
    _, h_ref = O.fit(cfg, p0, x.astype(np.float64), y.astype(np.float64), loss=O.LOSS_BCE_LOGITS, epochs=4,
                     batch_size=128, lr=1e-3, eps_fn=eps_fn, perm_fn=lambda e, n: perms[e],
                     beta_fn=lambda e: O.beta_schedule(e, 1e-3, 1e-1, 1, 3),
                     validation_data=(x[:256].astype(np.float64), y[:256].astype(np.float64)))
    assert set(hist) == set(h_ref)
    worst = {}
    for k in h_ref:
        a, b = np.asarray(hist[k], np.float64), np.asarray(h_ref[k], np.float64)
        worst[k] = float(np.max(np.abs(a - b) / (np.abs(b) + 1e-4)))
        if "accuracy" in k:
            np.testing.assert_allclose(a, b, atol=3e-2, err_msg=k)
        else:
            np.testing.assert_allclose(a, b, rtol=3e-2, atol=1e-4, err_msg=k)
    print("fit trajectory: worst relative deviation per series:", {k: round(v, 5) for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:6]})
    assert hist["loss"][-1] < hist["loss"][0]                                    # and it trains


def test_fp16_mode_range_edges():
    """(a) inputs out to |x| = 6 and log-variances near +-10 (sigma^2 from 4.5e-5 to 2.2e4) stay inside fp16 and match
    the fp32 path; (b) activations beyond fp16's 65 504 SATURATE (finite results, no inf/NaN) in 'fp16' mode -- the
    documented limit of the mode -- while 'bf16' and 'tf32' (8-bit exponents) still track the fp32 path."""
    cfg = _c0()
    B = 4096
    rng = np.random.default_rng(7)
    x = (rng.uniform(-6, 6, size=(B, 16))).astype(np.float32)
    y = (x[:, 0] * x[:, 1] > 0).astype(np.float32)[:, None]
    p = O.glorot_uniform_params(cfg, rng)
    encs, _ = O.unflatten(cfg, p)                                               # views into p
    for f in range(16):
        b2 = encs[f][-1][1]
        b2[32:] = np.where(np.arange(32) % 2 == 0, 10.0, -10.0) * (0.9 + 0.1 * rng.random(32))
    res = {}
    for prec in ("fp32", "fp16"):
        m = build_model(cfg, precision=prec)
        m.set_flat_weights(p)
        m.beta.assign(0.01)
        g, st = m.compute_gradients(x, y, step=1)
        res[prec] = (g.cpu().numpy(), st.cpu().numpy())
    assert np.isfinite(res["fp16"][0]).all() and np.isfinite(res["fp16"][1]).all()
    assert res["fp32"][1][:16].min() / B > 1000.0                               # the KLs really are in the e^10 regime
    np.testing.assert_allclose(res["fp16"][1], res["fp32"][1], rtol=5e-3)
    assert rel_err(res["fp16"][0], res["fp32"][0]) < 5e-3
    # (b) hidden activations ~ 2e5: scale the first encoder layer
    p_big = p.copy()
    encs, _ = O.unflatten(cfg, p_big)
    for f in range(16):
        encs[f][0][0][:] *= 4.0e4
        encs[f][-1][1][32:] = -1.0
        encs[f][1][0][:] *= 1e-3                                                # keep the later layers O(1) in exact arithmetic
    out = {}
    for prec in ("fp32", "fp16", "bf16", "tf32"):
        m = build_model(cfg, precision=prec)
        m.set_flat_weights(p_big)
        m.beta.assign(0.01)
        pred = np.asarray(m(x, step=1))
        g, st = m.compute_gradients(x, y, step=1)
        out[prec] = (pred, g.cpu().numpy(), st.cpu().numpy())
        assert np.isfinite(pred).all() and np.isfinite(out[prec][1]).all() and np.isfinite(out[prec][2]).all(), prec
    # 16 features x three layers of 11-bit (tf32) / 8-bit (bf16) operands at these magnitudes: 4x the per-step bounds
    assert rel_err(out["tf32"][0], out["fp32"][0]) < 2e-2
    assert rel_err(out["bf16"][0], out["fp32"][0]) < 1.6e-1
    assert rel_err(out["fp16"][0], out["fp32"][0]) > 5e-2                        # clamped at 65 504: visibly different, by design


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


_WORKER = r"""
import os, sys, json
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["DIB_ROOT"])
import dib_b200
from oracle import dib_oracle as O
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
x, y = O.boolean_circuit_truth_table()
m = dib_b200.DistributedIBNet([1] * 10, [128, 128], [256], 1, precision=os.environ["DIB_PREC"], seed=4)
m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
m.noise_seed = 99
h = m.fit(x, y, epochs=3, batch_size=256, shuffle=True, verbose=False, validation_data=(x[:256], y[:256]),
          callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)]).history
if rank == 0:
    np.savez(os.environ["DIB_OUT"], params=m.get_flat_weights(), **{k: np.asarray(v) for k, v in h.items()})
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.parametrize("prec", ["fp16", "fp32"])
def test_two_gpu_fit_equals_one_gpu_fit(tmp_path, prec):
    """On-hardware N-GPU == 1-GPU: `fit` over NCCL on 2 GPUs (rows of every global batch split between the ranks, one
    all-reduce of [grads || stats] per step) reproduces the single-GPU history and final weights."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    outs = {}
    for world in (1, 2):
        out = str(tmp_path / f"w{world}.npz")
        env = dict(os.environ, DIB_ROOT=ROOT, DIB_OUT=out, DIB_PREC=prec, MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(_free_port()), WORLD_SIZE=str(world))
        procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)))
                 for r in range(world)]
        for pr in procs:
            assert pr.wait(timeout=600) == 0
        outs[world] = np.load(out)
    a, b = outs[1], outs[2]
    assert set(a.files) == set(b.files)
    # Per-sample arithmetic is identical on 1 and 2 GPUs (noise keyed by the global row, same loss scale); what differs is the
    # fp32 summation grouping of the weight gradients (one register accumulator over all tiles vs. one per rank + NCCL sum), a
    # ~1e-7 relative perturbation that Adam's normalisation amplifies over the 12 steps -- more in the fp16 mode (long
    # in-register sums) than in the fp32 mode (32-row split partials on both sides).
    tol_p, tol_h = (5e-3, 2e-3) if prec == "fp16" else (2e-4, 2e-4)
    for k in a.files:
        if k == "params":
            assert rel_err(b[k], a[k]) < tol_p
        else:
            np.testing.assert_allclose(b[k], a[k], rtol=tol_h, atol=1e-5, err_msg=k)


@pytest.mark.parametrize("prec", ["fp16", "fp32"])
def test_cuda_graph_replay_is_bit_identical_to_eager(prec):
    """`fit` with the step replayed from CUDA graphs (device-resident Philox / Adam step counters) reproduces the
    eager-launch history and weights bit for bit."""
    import dib_b200
    x, y, cfg = _fit_case()
    res = {}
    for graph in (False, True):
        m = build_model(cfg, precision=prec, lr=1e-3, seed=4)
        m.use_cuda_graph = graph
        m.noise_seed = 7
        h = m.fit(x, y, epochs=3, batch_size=200, shuffle=True, verbose=False, validation_data=(x[:256], y[:256]),
                  callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)]).history
        if graph:
            assert len(m._graphs) >= 1 and m._replayed_launches > 0 and not m._graph_failed      # the graphs really replayed
        res[graph] = (h, m.get_flat_weights())
    assert set(res[True][0]) == set(res[False][0])
    for k in res[False][0]:
        np.testing.assert_array_equal(np.asarray(res[True][0][k]), np.asarray(res[False][0][k]), err_msg=k)
    np.testing.assert_array_equal(res[True][1], res[False][1])


@pytest.mark.gpu
def test_fp16_mode_batch_split_boundaries():
    """Weight-gradient kernels split the batch into slices of whole k-blocks (64 rows for the 16-bit kernels): batch sizes whose
    ceil(n / 32) is an odd multiple of 32 (20 557 -> 672-row slices before the fix) double-counted the 32 rows after every slice
    boundary in the integration network's weight gradients.  fp16 mode against the fp32 path, per variable."""
    import dib_b200
    from tests.test_gpu_parity import build_model, rel_err
    from oracle import dib_oracle as O
    cfg = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    rng = np.random.default_rng(77)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    for B in (20557, 19203):
        x = rng.standard_normal((B, 16)).astype(np.float32)
        y = (x[:, :1] * x[:, 1:2] > 0).astype(np.float32)
        g = {}
        for prec in ("fp32", "fp16"):
            m = build_model(cfg, precision=prec)
            m.set_flat_weights(p)
            m.beta.assign(0.02)
            gg, st = m.compute_gradients(x, y, step=3)
            g[prec] = gg.cpu().numpy()
        assert rel_err(g["fp16"], g["fp32"]) < 5e-3
        layout = m.param_layout() if hasattr(m, "param_layout") else None
        # per-variable check on the integration network's kernels (the last 2 x 3 variables of the flat vector)
        off = 0
        for v in m.trainable_variables:
            n = int(np.prod(v.shape))
            a, b = g["fp16"][off:off + n], g["fp32"][off:off + n]
            if np.abs(b).max() > 0:
                assert np.abs(a - b).max() / np.abs(b).max() < 2e-2, (v.name if hasattr(v, "name") else off)
            off += n
