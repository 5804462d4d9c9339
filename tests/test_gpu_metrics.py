"""GPU (H100): compiled Keras metrics (compile(metrics=, weighted_metrics=)) -- the metric tail of the statistics vector that
dib_metrics.cu reduces from the step's own outputs -- against the float64 metric oracle (tests/metrics_oracle.py), and the
rest of the step bit for bit against the same model without metrics on every loss site."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests import metrics_oracle as MO
from tests.test_gpu_fused16_vs_rounding_oracle import _c, _data, _expect_route, _params
from tests.test_gpu_parity import build_model
from tests.test_gpu_sample_weights import _weights

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _all_metrics(loss, probs=False):
    """(metrics, weighted_metrics): every metric the compiled loss admits."""
    from dib_b200 import metrics as M
    if loss == "sparse_ce_logits":
        return (["accuracy", "sparse_categorical_accuracy", "sparse_categorical_crossentropy",
                 M.SparseCategoricalCrossentropy(from_logits=True, name="sce_logits")],
                ["accuracy", "sparse_categorical_crossentropy"])
    if loss == "mse":
        return ["accuracy", "mse", "mae", "binary_accuracy", M.MeanSquaredError()], ["mae", M.BinaryAccuracy(threshold=0.2)]
    conf = ([M.AUC(), M.AUC(curve="PR", name="pr_auc"), M.Precision(), M.Recall(thresholds=0.3)] if probs else
            [M.AUC(from_logits=True), M.AUC(curve="PR", from_logits=True, name="pr_auc")])
    return (["accuracy", "binary_accuracy", "mse", "mae", "binary_crossentropy",
             M.BinaryCrossentropy(from_logits=not probs, name="bce")] + conf,
            ["mse", M.AUC(from_logits=not probs, num_thresholds=57), "accuracy"] + ([M.Precision(0.7)] if probs else []))


def _model16(cfg, prec, loss, metrics=None, weighted=None, mask=0, seed=0):
    import dib_b200
    m = dib_b200.DistributedIBNet(
        cfg.feature_dimensionalities, cfg.feature_encoder_architecture, cfg.integration_network_architecture,
        cfg.output_dimensionality, use_positional_encoding=cfg.use_positional_encoding,
        number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies, activation_fn=cfg.activation_fn,
        feature_embedding_dimension=cfg.feature_embedding_dimension, output_activation_fn=cfg.output_activation_fn,
        precision=prec, seed=seed)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=loss, metrics=metrics, weighted_metrics=weighted)
    m.debug_force_unfused(mask)
    return m


# loss site: (cfg kwargs, loss, precision, route of _expect_route or None for fp32 / tf32)
SITES = {
    "c0_fp16_fused_tail": (dict(F=16), "bce_logits", "fp16", "dgrad"),
    "c0_bf16_fused_tail": (dict(F=16), "bce_logits", "bf16", "dgrad"),
    "c0_fp16_probs_fused_tail": (dict(F=12, probs=True), "bce_probs", "fp16", "dgrad"),
    "head1_fp16": (dict(F=16, integ=(128, 256)), "bce_logits", "fp16", None),
    "head3_fp16_sce": (dict(F=16, out=3), "sparse_ce_logits", "fp16", None),
    "head6_bf16_mse": (dict(F=16, out=6), "mse", "bf16", None),
    "loss_kernel_fp32": (dict(F=6, out=3, integ=(64, 32)), "sparse_ce_logits", "fp32", None),
    "loss_kernel_tf32": (dict(F=6, integ=(64, 32), probs=True), "bce_probs", "tf32", None),
    "loss_kernel_fp32_mse6": (dict(F=4, out=6, integ=(64, 32)), "mse", "fp32", None),
}


@pytest.mark.parametrize("site", list(SITES))
def test_metrics_do_not_touch_training(site):
    """Gradients, the F + 3 statistics, fit history (loss, KL, accuracy) and final weights are bit-identical with and without
    compiled metrics; the metrics add one launch per step and their tail to dib_stats_count."""
    import dib_b200
    kw, loss, prec, route = SITES[site]
    cfg = _c(**kw)
    lid = {"bce_logits": O.LOSS_BCE_LOGITS, "bce_probs": O.LOSS_BCE_LOGITS, "sparse_ce_logits": O.LOSS_SPARSE_CE_LOGITS,
           "mse": O.LOSS_MSE}[loss]
    n = 128 * 9 + 5
    x, y, eps = _data(cfg, lid, n, 2)
    w = _weights(n, 2)
    mets, wmets = _all_metrics(loss, probs=cfg.output_activation_fn == "sigmoid")
    res = {}
    for with_metrics in (False, True):
        m = _model16(cfg, prec, loss, *((mets, wmets) if with_metrics else (["accuracy"], None)), seed=3)
        if route is not None or prec in ("fp16", "bf16"):
            _expect_route(m, prec, n, route)
        m.set_flat_weights(_params(cfg, 2))
        m.beta.assign(0.01)
        m._ensure_handle(n)
        F = cfg.number_features
        count = int(m._lib.dib_stats_count(m._handle))
        assert count == F + 3 + m._tail_len and (m._tail_len > 0) == with_metrics
        l0 = int(m._lib.dib_launch_count())
        g, st = m.compute_gradients(x, y, eps=eps, sample_weight=w)
        launches = int(m._lib.dib_launch_count()) - l0
        g, st = g.cpu().numpy(), st.cpu().numpy()
        h = m.fit(x, y, sample_weight=w, batch_size=256, epochs=2, verbose=False, validation_data=(x[:300], y[:300], w[:300]),
                  callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 1)]).history
        res[with_metrics] = (g, st[:F + 3], h, m.get_flat_weights(), launches, st[F + 3:])
    (g0, s0, h0, p0, l0), (g1, s1, h1, p1, l1) = res[False][:5], res[True][:5]
    assert np.array_equal(g0, g1) and np.array_equal(s0, s1)
    assert np.array_equal(p0, p1)
    for k, v in h0.items():
        assert h1[k] == v, k
    extra = [k for k in h1 if k not in h0]
    assert extra and all(np.isfinite(h1[k]).all() for k in extra), extra
    assert l1 == l0 + 1, (l0, l1)                                             # the metric kernel, and nothing else
    assert np.isfinite(res[True][5]).all()


def _st_model(varlen, metrics, weighted):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(2, [32], bottleneck_dimension=8, number_particles=12, key_dim=8, number_heads=2,
                                     number_attention_blocks=1, final_processing_arch=[16], seed=1, variable_set_sizes=varlen)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=metrics, weighted_metrics=weighted)
    return m


@pytest.mark.parametrize("varlen", [False, True])
def test_set_transformer_metrics_do_not_touch_training_and_count_sets(varlen):
    from dib_b200 import metrics as M
    rng = np.random.default_rng(5)
    n = 70
    xs = rng.standard_normal((n, 12, 2)).astype(np.float32)
    y = rng.integers(0, 2, (n, 1)).astype(np.float32)
    sizes = rng.integers(1, 13, n).astype(np.int32)
    x = (xs, sizes) if varlen else xs
    w = rng.uniform(0, 5, n).astype(np.float32)
    mets, wmets = _all_metrics("bce_logits")
    out = {}
    for with_metrics in (False, True):
        m = _st_model(varlen, *((mets, wmets) if with_metrics else (["accuracy"], None)))
        g, st = m.compute_gradients(x, y, sample_weight=w)
        h = m.fit(x, y, sample_weight=w, batch_size=32, epochs=2, verbose=False).history
        out[with_metrics] = (g.cpu().numpy(), st.cpu().numpy(), h, m.get_flat_weights(), m)
    F = 1
    assert np.array_equal(out[False][0], out[True][0]) and np.array_equal(out[False][1], out[True][1][:F + 3])
    assert np.array_equal(out[False][3], out[True][3])
    assert all(out[True][2][k] == v for k, v in out[False][2].items())
    # one row per set: the tail's weight sums count sets
    m = out[True][4]
    e = {x.name: x for x in m._metric_entries}
    st = out[True][1]
    assert st[F + 3 + e["mse"].offset + 1] == n
    np.testing.assert_allclose(st[F + 3 + e["weighted_mse"].offset + 1], w.astype(np.float64).sum(), rtol=1e-6)
    # kernel vs oracle on the sets' predictions
    xd, sd = m._inputs(x)
    yd = m._targets(y)
    wd = torch.from_numpy(w).cuda()
    z, _, st = m._forward(xd, yd, None, 7, 0, sizes=sd, weights=wd)
    vals = M.metric_values(m._metric_entries, st[F + 3:].cpu().numpy())
    z = z.cpu().numpy().astype(np.float64)
    for en in m._metric_entries:
        if en.in_tail and en.metric.kind != "confusion":
            ref = MO.for_metric(en.metric)
            ref.update(z, y, w if en.weighted else None)
            np.testing.assert_allclose(vals[en.name], ref.result(), rtol=1e-6, err_msg=en.name)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel against the oracle, on the step's own outputs
# ---------------------------------------------------------------------------------------------------------------------
KCASES = {
    "bce_logits": (O.DIBConfig([1, 2, 1, 3], [32, 32], [64, 32], 1, feature_embedding_dimension=8), "bce_logits"),
    "bce_probs": (O.DIBConfig([1, 2, 1, 3], [32, 32], [64, 32], 1, feature_embedding_dimension=8,
                              output_activation_fn="sigmoid"), "bce_probs"),
    "sce3": (O.DIBConfig([1, 2, 1, 3], [32, 32], [64, 32], 3, feature_embedding_dimension=8), "sparse_ce_logits"),
    "mse6": (O.DIBConfig([1, 2, 1, 3], [32, 32], [64, 32], 6, feature_embedding_dimension=8), "mse"),
}


def _near_threshold(p, thresholds, ulps=2):
    """Rows whose float32 p lies within `ulps` float32 ulps of a threshold (the fp32 sigmoid may put them either side)."""
    p32 = np.asarray(p, np.float32).reshape(-1, 1)
    t = np.asarray(thresholds, np.float32).reshape(1, -1)
    ulp = np.spacing(np.maximum(np.abs(p32), np.abs(t))).astype(np.float64)
    return (np.abs(p32.astype(np.float64) - t.astype(np.float64)) <= ulps * ulp).any(axis=1)


@pytest.mark.parametrize("n", [127, 4173])
@pytest.mark.parametrize("case", list(KCASES))
def test_metric_tail_matches_oracle_on_the_steps_outputs(case, n):
    from dib_b200 import metrics as M
    cfg, loss = KCASES[case]
    lid = {"bce_logits": O.LOSS_BCE_LOGITS, "bce_probs": O.LOSS_BCE_LOGITS, "sparse_ce_logits": O.LOSS_SPARSE_CE_LOGITS,
           "mse": O.LOSS_MSE}[loss]
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 7)).astype(np.float32)
    from tests.test_gpu_parity import make_labels
    y = make_labels(rng, lid, n, cfg.output_dimensionality)
    w = _weights(n, n)
    mets, wmets = _all_metrics(loss, probs=loss == "bce_probs")
    m = build_model(cfg, loss=loss)
    m.compile(optimizer="adam", loss=loss, metrics=mets, weighted_metrics=wmets)
    m.set_flat_weights(O.glorot_uniform_params(cfg, rng))
    xd, yd, wd = m._to_device(x), m._targets(y), torch.from_numpy(w).cuda()
    z, _, st = m._forward(xd, yd, None, 11, 0, weights=wd)
    st2 = m._forward(xd, yd, None, 11, 0, want_pred=False, weights=wd)[2]          # the tail from the workspace copy of z
    assert torch.equal(st, st2)
    F = cfg.number_features
    tail = st[F + 3:].cpu().numpy().astype(np.float64)
    z = z.cpu().numpy().astype(np.float64)
    vals = M.metric_values(m._metric_entries, tail)
    for e in m._metric_entries:
        if not e.in_tail:
            continue
        we = w if e.weighted else None
        mm = e.metric
        if mm.kind != "confusion":
            ref = MO.for_metric(mm)
            ref.update(z, y, we)
            np.testing.assert_allclose(vals[e.name], ref.result(), rtol=1e-6, atol=1e-7, err_msg=e.name)
            continue
        T = mm.num_thresholds
        thr = MO.auc_thresholds(T) if T > 1 else np.asarray([np.float32(mm.threshold)], np.float64)
        p = MO.sigmoid(z[:, 0]) if mm.from_logits else z[:, 0]
        b = (p[:, None] > thr[None, :]).sum(1)
        wr = np.ones(n) if we is None else we.astype(np.float64)
        pos = y[:, 0] != 0
        host = np.r_[np.bincount(b[~pos], wr[~pos], minlength=T + 1), np.bincount(b[pos], wr[pos], minlength=T + 1)]
        dev = tail[e.offset:e.offset + e.size]
        near = _near_threshold(p, thr) if mm.from_logits else np.zeros(n, bool)
        moved = np.abs(dev - host).sum()
        print(f"[metrics] {case} n={n} {e.name}: {int(near.sum())} rows within 2 ulp of a threshold, moved weight {moved:.3g}")
        # a row next to a threshold moves its weight between two buckets; weighted buckets are float32 sums besides
        assert moved <= 2 * wr[near].sum() * (1 + 1e-6) + (1e-6 * wr.sum() if we is not None else 0.0), e.name
        if not near.any():
            if we is None:
                assert np.array_equal(dev, host), e.name                   # counts: exact
            np.testing.assert_allclose(dev, host, rtol=1e-6, atol=1e-6 * wr.max(), err_msg=e.name)
            ref = MO.for_metric(mm)
            ref.update(z, y, we)
            np.testing.assert_allclose(vals[e.name], ref.result(), rtol=1e-6, atol=1e-7, err_msg=e.name)
    # repeated calls: bit-identical (fixed-order reductions, no float atomics)
    for _ in range(3):
        assert torch.equal(m._forward(xd, yd, None, 11, 0, weights=wd)[2], st)


# ---------------------------------------------------------------------------------------------------------------------
# fit / evaluate against the oracle fed the same batches' outputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_fit_and_evaluate_metric_histories_match_oracle(prec):
    import dib_b200
    from dib_b200 import metrics as M
    from tests.test_gpu_benched_mode import _fit_case
    x, y, cfg = _fit_case()
    rng = np.random.default_rng(1)
    sw = rng.uniform(0, 2, len(x)).astype(np.float32)
    xv, yv, wv = x[:256], y[:256], rng.uniform(0, 3, 256).astype(np.float32)
    mets = ["accuracy", "mse", M.BinaryCrossentropy(from_logits=True), M.AUC(from_logits=True)]
    wmets = [M.AUC(from_logits=True), "binary_accuracy"]
    cb = lambda: [dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 2)]

    def model():
        m = build_model(cfg, precision=prec, lr=1e-3, seed=4)
        m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=mets, weighted_metrics=wmets)
        m.noise_seed = 99
        return m
    m = model()
    h = m.fit(x, y, sample_weight=sw, epochs=3, batch_size=128, verbose=False, validation_data=(xv, yv, wv), callbacks=cb()).history
    names = [e.name for e in m._metric_entries]
    assert names == ["accuracy", "mse", "binary_crossentropy", "auc", "weighted_auc", "binary_accuracy"]
    assert set(h) == {"loss", "beta", "KL" + "0"} | {f"KL{i}" for i in range(10)} | set(names) | {
        "val_" + k for k in ["loss", "beta"] + [f"KL{i}" for i in range(10)] + names}
    # the oracle: a twin stepping through the same batches, metrics of each batch's outputs before its step
    r = model()
    ents = [e for e in r._metric_entries if e.in_tail]
    hist = {k: [] for k in [e.name for e in ents] + ["val_" + e.name for e in ents]}
    tol = 2e-3 if prec == "fp32" else 3e-2
    for epoch in range(3):
        r.beta.assign(O.beta_schedule(epoch, 1e-3, 1e-1, 1, 2))
        order = r.epoch_permutation(epoch, len(x)).cpu().numpy()
        acc = {e.name: MO.for_metric(e.metric) for e in ents}
        for b0 in range(0, len(x), 128):
            idx = order[b0:b0 + 128]
            xb, yb = r._to_device(x[idx]), r._targets(y[idx])
            z = r._forward(xb, yb, None, r._train_step_count, 0)[0].cpu().numpy().astype(np.float64)
            for e in ents:
                acc[e.name].update(z, y[idx], sw[idx] if e.weighted else None)
            r.train_on_batch(x[idx], y[idx], sample_weight=sw[idx])
        for e in ents:
            hist[e.name].append(acc[e.name].result())
        vacc = {e.name: MO.for_metric(e.metric) for e in ents}
        for b0 in range(0, 256, 128):
            z = r._forward(r._to_device(xv[b0:b0 + 128]), r._targets(yv[b0:b0 + 128]), None, 2 ** 31 + epoch, b0)[0]
            for e in ents:
                vacc[e.name].update(z.cpu().numpy().astype(np.float64), yv[b0:b0 + 128], wv[b0:b0 + 128] if e.weighted else None)
        for e in ents:
            hist["val_" + e.name].append(vacc[e.name].result())
    for k, ref in hist.items():
        np.testing.assert_allclose(h[k], ref, rtol=tol, atol=1e-4 if "accuracy" not in k else 1e-2, err_msg=k)
    # evaluate: [loss, *metrics, *weighted_metrics] in compile order
    d = m.evaluate(xv, yv, batch_size=128, sample_weight=wv)
    m._inference_calls -= 1
    lst = m.evaluate(xv, yv, batch_size=128, sample_weight=wv, return_dict=False)
    assert lst == [d["loss"]] + [d[k] for k in names]


# ---------------------------------------------------------------------------------------------------------------------
# graph replay, data parallelism, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_graph_replay_with_metrics_and_changing_weights_equals_eager():
    from tests.test_gpu_benched_mode import _c0, _c0_batch
    cfg = _c0()
    x, y = _c0_batch(512, 3)
    rng = np.random.default_rng(3)
    ws = [rng.uniform(0, 5, 512).astype(np.float32) for _ in range(7)]
    mets, wmets = _all_metrics("bce_logits")
    out = {}
    for graphs in (True, False):
        m = build_model(cfg, precision="fp16", seed=2)
        m.compile(optimizer="adam", loss="bce_logits", metrics=mets, weighted_metrics=wmets)
        m.use_cuda_graph = graphs
        res = [m.train_on_batch(x, y, sample_weight=w) for w in ws]
        res.append(m.train_on_batch(x, y))
        res += [m.train_on_batch(x, y, sample_weight=w, sync=False).get() for w in ws[:3]]
        out[graphs] = (res, m.get_flat_weights())
        if graphs:
            assert m._graphs and all(k[-2] for k in m._graphs), list(m._graphs)      # the metrics are in the key
    assert out[True][0] == out[False][0] and np.array_equal(out[True][1], out[False][1])
    assert "auc" in out[True][0][0] and "weighted_auc" in out[True][0][0]


_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["DIB_ROOT"])
import dib_b200
from dib_b200 import metrics as M
from tests.test_gpu_benched_mode import _fit_case
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(0)
if world > 1:
    dist.init_process_group("gloo")
x, y, cfg = _fit_case()
m = dib_b200.DistributedIBNet(cfg.feature_dimensionalities, cfg.feature_encoder_architecture,
                              cfg.integration_network_architecture, 1, precision=os.environ["DIB_PREC"], seed=4)
m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=["accuracy", "mse", M.AUC(from_logits=True)],
          weighted_metrics=[M.AUC(from_logits=True, curve="PR"), "binary_crossentropy"])
m.noise_seed = 99
rng = np.random.default_rng(0)
sw = rng.integers(0, 4, len(x)).astype(np.float32)
wv = rng.uniform(0, 3, 256).astype(np.float32)
lo, hi = rank * 128 // world, (rank + 1) * 128 // world
m.train_on_batch(x[lo:hi], y[lo:hi], sample_weight=sw[lo:hi])        # one step from the same weights: the summed tail
F = cfg.number_features
tail = m._gradstats[m._P + F + 3:].cpu().numpy()
h = m.fit(x, y, epochs=3, batch_size=128, verbose=False, sample_weight=sw, validation_data=(x[:256], y[:256], wv)).history
if rank == 0:
    np.savez(os.environ["DIB_OUT"], params=m.get_flat_weights(), graphs=len(m._graphs), tail=tail,
             **{k: np.asarray(v) for k, v in h.items()})
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_two_process_gloo_fit_with_metrics_equals_one_process_fit(tmp_path, prec):
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
    # the first step's tail: confusion counts (integer weights) exactly equal; the mean sums to float32 regrouping
    a, b = res[1].pop("tail"), res[2].pop("tail")
    conf = np.arange(2, 2 + 2 * 402)                 # the tail: mse [0, 2), auc [2, 404), weighted PR auc [404, 806), bce
    assert np.array_equal(a[conf], b[conf])
    np.testing.assert_allclose(b, a, rtol=1e-5)
    # counts of rows next to a threshold may move by the ~1e-7 regrouping of later steps: those histories get the accuracy bound
    loose = [k for k in res[1] if any(s in k for s in ("accuracy", "auc"))]
    for k in loose:
        np.testing.assert_allclose(res[2][k], res[1][k], atol=3e-2 if prec == "fp16" else 1e-2, err_msg=k)
    _compare_fits(*({k: v for k, v in r.items() if k not in loose} for r in (res[1], res[2])), prec)


def test_model_level_refusals():
    import dib_b200
    from dib_b200 import metrics as M
    from tests.test_gpu_benched_mode import _c0
    m = build_model(_c0())
    for bad in ([M.AUC()], [M.Precision()], ["f1"], [lambda a, b: a]):
        with pytest.raises(ValueError):
            m.compile(optimizer="adam", loss="bce_logits", metrics=bad)
    assert m.compiled_metrics_names == ["accuracy"] and m._tail_len == 0           # a refused compile changes nothing
    with pytest.raises(ValueError, match="InfoNCE"):
        m.compile(optimizer="adam", loss=dib_b200.losses.InfoNCE(4), weighted_metrics=["mse"])
    with pytest.raises(ValueError):
        m.compile(optimizer="adam", loss="external", metrics=["mse"])
    m.compile(optimizer="adam", loss="bce_logits", metrics=[M.AUC(from_logits=True)])
    x = np.zeros((8, 16), np.float32)
    with pytest.raises(ValueError, match="encoder-only"):
        m.encode(x)
    with pytest.raises(ValueError, match="encoder-only"):
        m.encoder_gradients(x, np.zeros((8, 16 * 32), np.float32))
    m.compile(optimizer="adam", loss="bce_logits", metrics=["accuracy"])           # back to no tail: the parent's stats row
    m._ensure_handle(8)
    assert int(m._lib.dib_stats_count(m._handle)) == 16 + 3 and m._gradstats.numel() == m._P + 19
    st = dib_b200.SetTransformerIBNet(2, [32], bottleneck_dimension=8, number_particles=12, key_dim=8, number_heads=2,
                                      number_attention_blocks=1, final_processing_arch=[16])
    with pytest.raises(ValueError, match="AUC\\(from_logits=True\\)"):
        st.compile(optimizer="adam", loss="bce_logits", metrics=[M.Recall()])
