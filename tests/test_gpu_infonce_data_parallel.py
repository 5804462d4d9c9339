"""GPU (H100): InfoNCE with global negatives on several ranks (losses.InfoNCE(..., negatives='global'), DESIGN.md section 7).

  * The three shard phases at one rank are dib_train_step bit for bit (the refactor behind them changed nothing).
  * R virtual ranks in one process -- R handles on one set of weights, the all-gathers done by writing into one e_all /
    lse_all -- give the one-rank lse_all bit for bit and the one-rank gradient up to the grouping of the weight-gradient sums.
  * fit on two processes (gloo on one GPU; NCCL on two GPUs when there are two) equals fit on one, and graph replay equals
    eager launches at world 2.

Tolerances, with what an H100 measured (NVIDIA H100 80GB HBM3):
  * virtual ranks, fp32: summed gradient vs the one-rank step 1e-5 max-norm relative (<= 3.1e-7 measured); vs the float64
    oracle 5e-5 overall and 2e-4 per variable (the bounds of test_gpu_infonce.py);
  * virtual ranks, tf32 / fp16 / bf16 vs the one-rank step of the same precision: 5e-3, the N-GPU bound of
    test_gpu_benched_mode.py (<= 4.4e-7 measured);
  * fit, world 2 vs world 1, 12 Adam steps: fp32 history 2e-4 and weights 2e-4 (<= 1e-7 and 9.4e-7 measured); fp16 history
    5e-3 and weights 1.5e-2 (2.3e-3 on KL0 and 8.9e-3 measured, the loss within 3e-6).  One step differs by ~1e-7 (the
    virtual-rank bound above); in fp16 that moves some 16-bit operand roundings by one ulp, and the InfoNCE gradient
    and Adam amplify it over the steps.
"""

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests import infonce_oracle as IO
from tests.gpu_cases import CFG, YARCH, YD, _compare_fits, data, params, rel_err, run_workers, temperature_of

pytestmark = pytest.mark.gpu
F = CFG.number_features


def global_negatives_model(similarity="l2", precision="fp32", seed=0, negatives="global"):
    import dib_b200
    m = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                                  CFG.integration_network_architecture, CFG.output_dimensionality, output_activation_fn=None,
                                  precision=precision, seed=seed)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.InfoNCE(YD, YARCH, similarity=similarity,
                                                                          temperature=temperature_of(similarity),
                                                                          negatives=negatives))
    return m


def shard_step(models, x, y, eps, step=0):
    """One train step of len(models) virtual ranks of the global batch (x, y, eps): phase 1 on every rank into one e_all,
    phase 2 into one lse_all, phase 3.  Returns (e_all, lse_all, [grads per rank], [stats per rank])."""
    R, n = len(models), x.shape[0]
    nl = n // R
    e_all, lse_all = models[0]._infonce_buffers(n)
    xs, ys, es = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, eps)]
    for r, m in enumerate(models):
        m._ensure_handle(nl)
        m._set_device_step(False)
        sl = slice(r * nl, (r + 1) * nl)
        m._infonce_forward(xs[sl], ys[sl], e_all, n, r * nl, es[sl].contiguous(), step, r * nl, training=True)
    for r, m in enumerate(models):
        m._infonce_lse(nl, e_all, lse_all, n, r * nl, m._gradstats[m._P:])
    grads, stats = [], []
    for r, m in enumerate(models):
        sl = slice(r * nl, (r + 1) * nl)
        m._infonce_backward(xs[sl], e_all, lse_all, n, r * nl, es[sl].contiguous(), step, r * nl)
        grads.append(m._gradstats[:m._P].clone())
        stats.append(m._gradstats[m._P:].clone())
    return e_all, lse_all, grads, stats


@pytest.mark.parametrize("n", [512, 4160])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_phases_at_one_rank_are_the_train_step_bit_for_bit(similarity, precision, n):
    m = global_negatives_model(similarity, precision)
    m.set_flat_weights(params(1))
    m.beta.assign(0.01)
    x, y, eps = data(n, 2)
    g, st = m.compute_gradients(x, y, eps=eps, step=5)
    _, _, g1, st1 = shard_step([m], x, y, eps, step=5)
    assert torch.equal(g1[0], g), (similarity, precision, n, (g1[0] - g).abs().max().item())
    assert torch.equal(st1[0], st)


def _virtual_ranks(similarity, precision, R, n=1024):
    p = params(3)
    x, y, eps = data(n, 4)
    ref = global_negatives_model(similarity, precision)
    ref.set_flat_weights(p)
    ref.beta.assign(0.01)
    g_ref, st_ref = ref.compute_gradients(x, y, eps=eps)
    models = []
    for _ in range(R):
        m = global_negatives_model(similarity, precision)
        m.set_flat_weights(p)
        m.beta.assign(0.01)
        models.append(m)
    e_all, lse_all, grads, stats = shard_step(models, x, y, eps)
    # the one-rank sweep of the same e_all: phase 1 sets up the workspace, then its e_all is replaced by the gathered one
    one = global_negatives_model(similarity, precision)
    one.set_flat_weights(p)
    e1_all, lse1_all = one._infonce_buffers(n)
    one._ensure_handle(n)
    one._infonce_forward(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), e1_all, n, 0,
                         torch.from_numpy(eps).cuda(), 0, 0, training=True)
    one._infonce_lse(n, e_all, lse1_all, n, 0, one._gradstats[one._P:])
    return p, (x, y, eps), (g_ref, st_ref), (e_all, lse_all, lse1_all, e1_all), (sum(grads), sum(stats))


@pytest.mark.parametrize("R", [2, 4, 8])
@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_virtual_ranks_fp32(similarity, R):
    p, (x, y, eps), (g_ref, st_ref), (e_all, lse_all, lse1_all, e1_all), (g, st) = _virtual_ranks(similarity, "fp32", R)
    assert torch.equal(lse_all, lse1_all), (lse_all - lse1_all).abs().max().item()
    print(f"{similarity} R={R}: e_all vs one-rank forward max |diff| {(e_all - e1_all).abs().max().item():.3g}")
    g, g_ref = g.cpu().numpy(), g_ref.cpu().numpy()
    e = rel_err(g, g_ref)
    print(f"{similarity} R={R}: summed gradient vs one-rank step {e:.3g}")
    assert e < 1e-5, e
    n = x.shape[0]
    st, st_ref = st.cpu().numpy(), st_ref.cpu().numpy()
    assert st[F + 2] == n and st[F + 1] == 0
    np.testing.assert_allclose(st, st_ref, rtol=1e-5)
    g64, loss64, kl64 = IO.infonce_train_grads(CFG, p, x, y, eps, 0.01, y_dimensionality=YD, y_encoder_architecture=YARCH,
                                               similarity=similarity, temperature=temperature_of(similarity))
    assert rel_err(g, g64) < 5e-5
    m = global_negatives_model(similarity)
    for i, v in enumerate(m.trainable_variables):
        off = m._var_off[i]
        assert rel_err(g[off:off + v.numel()], g64[off:off + v.numel()]) < 2e-4, (similarity, i)
    assert abs(st[F] / n - loss64) < 2e-5 * max(1.0, abs(loss64))


@pytest.mark.parametrize("R", [2, 8])
@pytest.mark.parametrize("precision", ["tf32", "fp16", "bf16"])
def test_virtual_ranks_tensor_core_precisions(precision, R):
    _, _, (g_ref, st_ref), (_, lse_all, lse1_all, _), (g, st) = _virtual_ranks("l2", precision, R)
    assert torch.equal(lse_all, lse1_all)
    e = rel_err(g.cpu().numpy(), g_ref.cpu().numpy())
    print(f"{precision} R={R}: summed gradient vs one-rank step {e:.3g}")
    assert e < 5e-3, e
    np.testing.assert_allclose(st.cpu().numpy(), st_ref.cpu().numpy(), rtol=5e-3)


def test_refusals_come_before_any_collective(monkeypatch):
    import dib_b200
    from dib_b200 import parallel

    def boom(*a, **k):
        raise AssertionError("a collective ran")
    x, y, _ = data(64, 5)
    plain = global_negatives_model(negatives=None)
    glob = global_negatives_model()
    monkeypatch.setattr(parallel, "all_gather_rows_", boom)
    monkeypatch.setattr(parallel, "allreduce_sum_", boom)
    monkeypatch.setattr(parallel, "world_and_rank", lambda group=None: (2, 0))
    for call in (lambda: plain.fit(x, y, batch_size=32, verbose=False), lambda: plain.evaluate(x, y, batch_size=32),
                 lambda: plain.train_on_batch(x[:32], y[:32]), lambda: plain.compute_gradients(x[:32], y[:32])):
        with pytest.raises(NotImplementedError, match="negatives='global'") as ei:
            call()
        assert "all-gather" in str(ei.value)
    with pytest.raises(NotImplementedError, match="all-gather"):
        plain.compile(loss=dib_b200.losses.InfoNCE(YD, YARCH))
    for call in (lambda: glob.fit(x, y, batch_size=31, verbose=False), lambda: glob.evaluate(x, y, batch_size=33)):
        with pytest.raises(ValueError, match="equal shards"):
            call()
    with pytest.raises(ValueError, match="equal shards"):
        glob.compute_gradients(x[:32], y[:32], global_batch=63)


def test_shard_entry_points_validate_their_arguments():
    from dib_b200 import _lib
    m = global_negatives_model()
    x, y, _ = data(64, 6)
    xs, ys = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    m._ensure_handle(64)
    e_all, lse_all = m._infonce_buffers(128)
    with pytest.raises(_lib.DibError, match="row_offset"):
        m._infonce_forward(xs, ys, e_all, 128, 100, None, 0, 0, training=True)
    with pytest.raises(_lib.DibError, match="max_batch"):
        m._infonce_lse(65, e_all, lse_all, 128, 0, m._gradstats[m._P:])
    with pytest.raises(_lib.DibError, match="16-byte"):
        m._infonce_lse(64, e_all.view(-1)[1:], lse_all, 128, 0, m._gradstats[m._P:])
    other = global_negatives_model()
    other.compile(loss="mse")
    other._ensure_handle(64)
    with pytest.raises(_lib.DibError, match="not DIB_LOSS_INFONCE"):
        other._infonce_lse(64, e_all, lse_all, 128, 0, other._gradstats[other._P:])


_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["DIB_ROOT"])
import dib_b200
from tests.gpu_cases import CFG, YD, YARCH, data
rank, world, backend = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), os.environ["DIB_BACKEND"]
dev = torch.device("cuda", rank if backend == "nccl" else 0)
torch.cuda.set_device(dev)
if world > 1:
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
n, nv = 1024, 300
x, y, _ = data(n + nv, 12)
m = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                              CFG.integration_network_architecture, CFG.output_dimensionality, output_activation_fn=None,
                              precision=os.environ["DIB_PREC"], seed=4)
m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.InfoNCE(YD, YARCH, negatives="global"))
m.noise_seed = 99
h = m.fit(x[:n], y[:n], epochs=3, batch_size=256, verbose=False, validation_data=(x[n:], y[n:]),
          callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)]).history
graphs = len(m._graphs)
if rank == 0:
    np.savez(os.environ["DIB_OUT"], params=m.get_flat_weights(), graphs=graphs, **{k: np.asarray(v) for k, v in h.items()})
if world > 1:
    dist.destroy_process_group()
"""


def _run_fit(tmp_path, world, prec, backend, graphs):
    return run_workers(tmp_path, _WORKER, world, str(tmp_path / f"w{world}_{prec}_{backend}_{int(graphs)}.npz"), DIB_PREC=prec,
                       DIB_BACKEND=backend, DIB_CUDA_GRAPH="auto" if graphs else "0")


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_two_process_gloo_fit_equals_one_process_fit(tmp_path, prec):
    """Two processes on the one GPU, exchanging over gloo: the data-parallel InfoNCE fit reproduces the one-process fit, and
    its graph-replayed run equals its eager run bit for bit."""
    one = _run_fit(tmp_path, 1, prec, "gloo", True)
    two = _run_fit(tmp_path, 2, prec, "gloo", True)
    two_eager = _run_fit(tmp_path, 2, prec, "gloo", False)
    assert int(two["graphs"]) > 0 and int(two_eager["graphs"]) == 0
    for k in two:
        if k != "graphs":
            np.testing.assert_array_equal(two[k], two_eager[k], err_msg=k)
    _compare_fits(one, two, prec)


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_two_gpu_nccl_fit_equals_one_gpu_fit(tmp_path, prec):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _compare_fits(_run_fit(tmp_path, 1, prec, "nccl", True), _run_fit(tmp_path, 2, prec, "nccl", True), prec)
