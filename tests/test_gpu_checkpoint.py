"""GPU (H100): checkpoints.  A run interrupted after epoch k and resumed from its backup in a fresh model object ends
bit-identical to the run that was never interrupted -- parameters, optimizer slots, optimizer step, Philox step count and the
history -- because every random draw is keyed by state the checkpoint holds.  Also: save_weights / load_weights across
precisions and into live CUDA graphs, load_model, the refusals, data-parallel resume and ModelCheckpoint(save_best_only).

The interruption is a plain Python exception raised by a callback listed after BackupAndRestore, at the end of epoch k."""
import os

import numpy as np
import pytest

from tests.gpu_cases import CFG, YARCH, YD, data, run_workers, set_transformer_model, small, varlen_set_case

pytestmark = pytest.mark.gpu


class _Stop(Exception):
    pass


def _recorder(stop_at=None):
    """A callback that records each epoch's logs (and a copy of the weights), then raises at the end of epoch ``stop_at``."""
    import dib_b200

    class Recorder(dib_b200.Callback):
        def __init__(self):
            self.logs, self.weights = [], []

        def on_epoch_end(self, epoch, logs=None):
            self.logs.append((epoch, dict(logs)))
            self.weights.append(self.model.get_flat_weights().copy())
            if epoch == stop_at:
                raise _Stop(epoch)

    return Recorder()


def _state(m):
    return dict(params=m._params.cpu().numpy().copy(), m=m._m.cpu().numpy().copy(), v=m._v.cpu().numpy().copy(),
                step=m._step_dev.cpu().numpy().copy(), count=np.int64(m._train_step_count))


def _assert_same_state(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def _c0_data(n=1024, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 16)).astype(np.float32)
    y = (x[:, 0] * x[:, 1] + np.sin(2 * x[:, 2]) + 0.5 * x[:, 3] > 0).astype(np.float32)[:, None]
    return x, y


def _c0_model(precision="fp32", seed=3, optimizer=None, metrics=("accuracy",)):
    import dib_b200
    m = dib_b200.DistributedIBNet([1] * 16, [128, 128], [256, 256], 1, precision=precision, seed=seed)
    m.compile(optimizer=optimizer or dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True),
              metrics=list(metrics))
    m.noise_seed = 11
    return m


def _fit_interrupted(build, fit_kw, epochs, stop_at, backup_dir, extra_callbacks=lambda: []):
    """(uninterrupted model, its records, extras) and (resumed model, first records + resumed records, extras of both)."""
    import dib_b200
    ref = build()
    rec, extra = _recorder(), extra_callbacks()
    ref.fit(epochs=epochs, verbose=False, callbacks=extra + [rec], **fit_kw)
    first = build()
    rec1, extra1 = _recorder(stop_at), extra_callbacks()
    with pytest.raises(_Stop):
        first.fit(epochs=epochs, verbose=False, callbacks=extra1 + [dib_b200.BackupAndRestore(backup_dir), rec1], **fit_kw)
    assert os.path.exists(os.path.join(backup_dir, "backup.npz"))           # the exception skipped on_train_end
    resumed = build()
    rec2, extra2 = _recorder(), extra_callbacks()
    resumed.fit(epochs=epochs, verbose=False, callbacks=extra2 + [dib_b200.BackupAndRestore(backup_dir), rec2], **fit_kw)
    assert not os.path.exists(os.path.join(backup_dir, "backup.npz"))       # delete_checkpoint at on_train_end
    assert [e for e, _ in rec2.logs] == list(range(stop_at + 1, epochs))
    return (ref, rec, extra), (resumed, rec1.logs + rec2.logs, (extra1, extra2))


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_plain_model_resumed_fit_is_bit_identical(tmp_path, precision):
    import dib_b200
    from dib_b200 import metrics as M
    x, y = _c0_data()
    xv, yv = _c0_data(256, 1)
    build = lambda: _c0_model(precision, metrics=["accuracy", M.AUC(from_logits=True)])
    extras = lambda: [dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 4),
                      dib_b200.InfoPerFeatureCallback(1, xv, evaluation_batch_size=128, number_evaluation_batches=2)]
    fit_kw = dict(x=x, y=y, batch_size=256, validation_data=(xv, yv))
    (ref, rec, extra), (res, logs, (extra1, extra2)) = _fit_interrupted(build, fit_kw, 6, 2, str(tmp_path / "bk"), extras)
    assert ref._graphs and res._graphs                                     # CUDA graphs were on
    _assert_same_state(_state(ref), _state(res))
    assert logs == rec.logs
    assert "auc" in logs[0][1] and "val_auc" in logs[0][1]
    assert extra1[1].bounds + extra2[1].bounds == extra[1].bounds
    assert res._epochs_done == 6 and res.beta.value() == ref.beta.value()


def _other_model(kind):
    """(build, fit kwargs) of the other model kinds, at small sizes."""
    import dib_b200
    if kind in ("sgd_nesterov", "rmsprop"):
        opt = (lambda: dib_b200.SGD(0.05, momentum=0.9, nesterov=True)) if kind == "sgd_nesterov" else \
              (lambda: dib_b200.RMSprop(1e-3, momentum=0.5))
        x, y = _c0_data(512)
        return (lambda: _c0_model("fp16", optimizer=opt())), dict(x=x, y=y, batch_size=128, validation_data=(x[:128], y[:128]))
    if kind == "infonce":
        x, y, _ = data(768, 12)

        def build():
            m = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                                          CFG.integration_network_architecture, CFG.output_dimensionality, seed=5)
            m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.InfoNCE(YD, YARCH, similarity="cosine",
                                                                                  temperature=0.5))
            return m
        return build, dict(x=x[:512], y=y[:512], batch_size=128, validation_data=(x[512:], y[512:]))
    variable = kind == "set_variable"
    cfg = small(12)
    sizes = np.random.default_rng(4).integers(1, 13, 96).astype(np.int32)
    _, xs, ys, _, sizes = varlen_set_case(cfg, sizes, 7)
    xin = (xs, sizes) if variable else xs
    return (lambda: set_transformer_model(cfg, seed=2, variable=variable, metrics=["accuracy"])), dict(x=xin, y=ys, batch_size=32)


@pytest.mark.parametrize("kind", ["sgd_nesterov", "rmsprop", "infonce", "set_fixed", "set_variable"])
def test_other_model_kinds_resumed_fit_is_bit_identical(tmp_path, kind):
    import dib_b200
    build, fit_kw = _other_model(kind)
    anneal = lambda: [dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-2, 1, 2)]
    (ref, rec, _), (res, logs, _) = _fit_interrupted(build, fit_kw, 4, 1, str(tmp_path / "bk"), anneal)
    _assert_same_state(_state(ref), _state(res))
    assert logs == rec.logs
    if kind == "infonce":
        assert res.output_encoder is not None and res._P > res._var_off[res._n_model_vars]
    if kind == "sgd_nesterov":
        assert np.abs(res._m.cpu().numpy()).max() > 0                      # the velocity is part of the state


def test_simple_encoder_train_on_batch_loop_continues_after_load_model(tmp_path):
    """nb-bool's custom loop: train_on_batch with beta set every step, model.save mid-loop, load_model, continue."""
    import dib_b200
    rng = np.random.default_rng(0)
    x = rng.choice([-1.0, 1.0], size=(1024, 10)).astype(np.float32)
    y = (x[:, :3].prod(1) > 0).astype(np.float32)[:, None]
    betas = np.logspace(-4, -1, 24).astype(np.float32)

    def build():
        m = dib_b200.DistributedIBNet([1] * 10, "simple", [64, 64], 1, feature_embedding_dimension=1, seed=8)
        m.compile(optimizer=dib_b200.Adam(3e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True))
        return m

    def steps(m, ks):
        out = []
        for k in ks:
            m.beta.assign(betas[k])
            b = (k * 128) % 1024
            out.append(m.train_on_batch(x[b:b + 128], y[b:b + 128]))
        return out

    ref = build()
    ref_out = steps(ref, range(24))
    first = build()
    out = steps(first, range(12))
    path = str(tmp_path / "loop.npz")
    first.save(path)
    del first
    loaded = dib_b200.models.load_model(path)
    out += steps(loaded, range(12, 24))
    assert out == ref_out
    _assert_same_state(_state(ref), _state(loaded))
    assert loaded._graphs


def test_weights_round_trip_and_predictions(tmp_path):
    import dib_b200
    x, y = _c0_data(512)
    m = _c0_model("fp32", seed=1)
    m.fit(x, y, epochs=1, batch_size=128, verbose=False)
    path = str(tmp_path / "w.npz")
    m.save_weights(path)
    with np.load(path, allow_pickle=False) as npz:                       # Keras orientation, readable without the engine
        assert npz["feature_encoder_0/dense_0/kernel"].shape == m.feature_encoders[0].get_weights()[0].shape
        assert npz["integration_network/dense_2/kernel"].shape == (256, 1)
        assert np.array_equal(npz["integration_network/dense_0/kernel"], m.integration_network.get_weights()[0])
    fresh = _c0_model("fp32", seed=9)
    assert not np.array_equal(fresh.get_flat_weights(), m.get_flat_weights())
    fresh.load_weights(path)
    assert np.array_equal(fresh.get_flat_weights(), m.get_flat_weights())
    eps = np.random.default_rng(2).standard_normal((64, 16, 32)).astype(np.float32)
    assert np.array_equal(fresh(x[:64], eps=eps), m(x[:64], eps=eps))
    # a model file carries the weights too
    m.save(str(tmp_path / "m.npz"))
    fresh2 = _c0_model("fp32", seed=10)
    fresh2.load_weights(str(tmp_path / "m.npz"))
    assert np.array_equal(fresh2.get_flat_weights(), m.get_flat_weights())


def test_fp32_file_into_fp16_model_equals_set_flat_weights(tmp_path):
    x, y = _c0_data(512)
    m = _c0_model("fp32", seed=1)
    m.fit(x, y, epochs=1, batch_size=128, verbose=False)
    path = str(tmp_path / "w.npz")
    m.save_weights(path)
    a, b = _c0_model("fp16", seed=4), _c0_model("fp16", seed=4)
    a.load_weights(path)
    b.set_flat_weights(m.get_flat_weights())
    assert np.array_equal(a.get_flat_weights(), b.get_flat_weights())
    assert [a.train_on_batch(x[:256], y[:256]) for _ in range(3)] == [b.train_on_batch(x[:256], y[:256]) for _ in range(3)]
    assert np.array_equal(a.get_flat_weights(), b.get_flat_weights())
    # and back: an fp16 model's file into an fp32 model
    a.save_weights(path)
    c = _c0_model("fp32", seed=6)
    c.load_weights(path)
    assert np.array_equal(c.get_flat_weights(), a.get_flat_weights())


def test_load_weights_into_captured_graphs(tmp_path):
    """Loading copies into the live parameter buffer: a model whose step is already captured trains on from the loaded
    weights exactly as the same model run eagerly."""
    x, y = _c0_data(512)
    src = _c0_model("fp16", seed=1)
    src.fit(x, y, epochs=1, batch_size=128, verbose=False)
    path = str(tmp_path / "w.npz")
    src.save_weights(path)
    outs = {}
    for graphs in (True, False):
        m = _c0_model("fp16", seed=7)
        m.use_cuda_graph = graphs
        before = [m.train_on_batch(x[:128], y[:128]) for _ in range(4)]
        if graphs:
            assert m._graphs                                                 # captured before the load
            replayed = m._replayed_launches
        m.load_weights(path)
        after = [m.train_on_batch(x[128:256], y[128:256]) for _ in range(3)]
        if graphs:
            assert m._replayed_launches > replayed and len(m._graphs) == 1   # replayed, not re-captured
        outs[graphs] = (before, after, _state(m))
    assert outs[True][0] == outs[False][0] and outs[True][1] == outs[False][1]
    _assert_same_state(outs[True][2], outs[False][2])


def test_load_model_restores_configuration_and_counters(tmp_path):
    import dib_b200
    from dib_b200 import metrics as M
    x, y = _c0_data(512)
    m = _c0_model("fp16", seed=1, metrics=["accuracy", "mse", M.AUC(from_logits=True, num_thresholds=57)])
    m.compile(optimizer=dib_b200.Adam(2e-3, beta_1=0.8), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True),
              metrics=["accuracy", "mse", M.AUC(from_logits=True, num_thresholds=57)],
              weighted_metrics=["accuracy", M.AUC(from_logits=True, curve="PR", name="pr")])
    m.fit(x, y, epochs=2, batch_size=128, verbose=False, sample_weight=np.linspace(0, 2, 512, dtype=np.float32))
    m.optimizer.learning_rate = 5e-4
    m.beta.assign(0.0125)
    m.predict(x[:64])
    path = str(tmp_path / "m.npz")
    m.save(path)
    ld = dib_b200.models.load_model(path)
    assert ld.precision == "fp16" and ld.kernel_info(256) == m.kernel_info(256)
    assert ld._loss_kind == m._loss_kind and ld.compiled_metrics_names == m.compiled_metrics_names
    assert [(e.name, e.weighted, e.in_tail and e.spec()) for e in ld._metric_entries] == \
           [(e.name, e.weighted, e.in_tail and e.spec()) for e in m._metric_entries]
    assert type(ld.optimizer) is dib_b200.Adam and ld.optimizer.beta_1 == 0.8 and ld.optimizer.learning_rate == 5e-4
    assert float(ld._lr_dev.item()) == float(np.float32(5e-4))
    assert (ld._train_step_count, ld._epochs_done, ld._inference_calls, ld.beta.value()) == \
           (m._train_step_count, 2, m._inference_calls, np.float32(0.0125))
    _assert_same_state(_state(m), _state(ld))
    assert m.evaluate(x, y, batch_size=128) == ld.evaluate(x, y, batch_size=128)
    assert m.train_on_batch(x[:128], y[:128]) == ld.train_on_batch(x[:128], y[:128])
    # without the optimizer: an uncompiled model with the weights
    m.save(path, include_optimizer=False)
    bare = dib_b200.models.load_model(path)
    assert bare.optimizer is None and np.array_equal(bare.get_flat_weights(), m.get_flat_weights())
    m.save_weights(path)
    with pytest.raises(ValueError, match="load_weights"):
        dib_b200.models.load_model(path)


def test_refused_restores_change_nothing(tmp_path):
    import dib_b200
    from dib_b200 import checkpoint
    x, y = _c0_data(512)
    src = _c0_model("fp32", seed=1)
    src.fit(x, y, epochs=1, batch_size=128, verbose=False)
    path = str(tmp_path / "m.npz")
    src.save(path)

    def counters(m):
        return m._epochs_done, m._inference_calls, m.noise_seed, m.seed, m.beta.value(), m._lr_host

    def refused(m, file, xb, yb, match, weights_match=None):
        m.train_on_batch(xb, yb)
        before, before_counters = _state(m), counters(m)
        with pytest.raises(ValueError, match=match):
            m._restore(*checkpoint.read(file))
        if weights_match:
            with pytest.raises(ValueError, match=weights_match):
                m.load_weights(file)
        _assert_same_state(before, _state(m))
        assert counters(m) == before_counters

    wider = dib_b200.DistributedIBNet([1] * 16, [128, 128], [256, 128], 1, seed=2)
    wider.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits")
    refused(wider, path, x[:128], y[:128], "architecture differs in 'integration_network_architecture'",
            r"variable \d+ differs: the file has 'integration_network/dense_1/kernel' \(256, 256\)")
    sgd = _c0_model("fp32", seed=2, optimizer=dib_b200.SGD(0.01))
    refused(sgd, path, x[:128], y[:128], "trained with Adam.*compiled with SGD")
    adam = _c0_model("fp32", seed=2, optimizer=dib_b200.Adam(1e-3, beta_2=0.99))
    refused(adam, path, x[:128], y[:128], "optimizer hyperparameters differ")

    def nce_model(temperature):
        m = dib_b200.DistributedIBNet(CFG.feature_dimensionalities, CFG.feature_encoder_architecture,
                                      CFG.integration_network_architecture, CFG.output_dimensionality, seed=5)
        m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.InfoNCE(YD, YARCH, temperature=temperature))
        return m
    xi, yi, _ = data(256, 3)
    a = nce_model(1.0)
    a.train_on_batch(xi[:128], yi[:128])
    nce_path = str(tmp_path / "nce.npz")
    a.save(nce_path)
    refused(nce_model(0.5), nce_path, xi[:128], yi[:128], "the loss differs")


_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["DIB_ROOT"])
import dib_b200
from dib_b200 import checkpoint
from tests.gpu_cases import _fit_case
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(0)
if world > 1:
    dist.init_process_group("gloo")
if rank != 0:
    def _refuse(*a, **k):
        raise AssertionError("only rank 0 writes checkpoints")
    checkpoint.write = _refuse
stop_at = int(os.environ["DIB_STOP"])


class Stop(dib_b200.Callback):
    history = {}

    def on_epoch_end(self, epoch, logs=None):
        for k, v in logs.items():
            self.history.setdefault(k, []).append(v)
        if epoch == stop_at:
            raise KeyboardInterrupt


x, y, cfg = _fit_case()
m = dib_b200.DistributedIBNet(cfg.feature_dimensionalities, cfg.feature_encoder_architecture,
                              cfg.integration_network_architecture, 1, precision="fp32", seed=4)
m.compile(optimizer=dib_b200.Adam(1e-3), loss="bce_logits", metrics=["accuracy"])
m.noise_seed = 99
cbs = [dib_b200.InfoBottleneckAnnealingCallback(1e-3, 1e-1, 1, 3)]
if os.environ["DIB_BACKUP"]:
    cbs.append(dib_b200.BackupAndRestore(os.environ["DIB_BACKUP"]))
cbs.append(Stop())
try:
    m.fit(x, y, epochs=5, batch_size=256, verbose=False, validation_data=(x[:256], y[:256]), callbacks=cbs)
except KeyboardInterrupt:
    pass
h = Stop.history
if rank == 0:
    np.savez(os.environ["DIB_OUT"], params=m.get_flat_weights(), m=m._m.cpu().numpy(), v=m._v.cpu().numpy(),
             step=m._step_dev.cpu().numpy(), count=m._train_step_count, **{k: np.asarray(v) for k, v in h.items()})
if world > 1:
    dist.destroy_process_group()
"""


def _run_workers(tmp_path, name, world, backup, stop_at=-1):
    return run_workers(tmp_path, _WORKER, world, str(tmp_path / f"{name}.npz"), DIB_BACKUP=backup, DIB_STOP=str(stop_at))


def _hist(r):
    return {k: v for k, v in r.items() if k not in ("params", "m", "v", "step", "count")}


def test_two_process_gloo_resume_is_bit_identical_and_one_process_state_resumes_on_two(tmp_path):
    full2 = _run_workers(tmp_path, "full2", 2, "")
    bk = str(tmp_path / "bk2")
    first2 = _run_workers(tmp_path, "first2", 2, bk, stop_at=1)
    assert os.path.exists(os.path.join(bk, "backup.npz"))
    resumed2 = _run_workers(tmp_path, "resumed2", 2, bk)
    for k in ("params", "m", "v", "step", "count"):
        assert np.array_equal(resumed2[k], full2[k]), k
    for k, v in _hist(full2).items():
        assert np.array_equal(np.concatenate([first2[k], resumed2[k]]), v), k
    # a state saved by one process continues on two: the saved state does not depend on the rank
    full1 = _run_workers(tmp_path, "full1", 1, "")
    bk1 = str(tmp_path / "bk1")
    _run_workers(tmp_path, "first1", 1, bk1, stop_at=1)
    resumed12 = _run_workers(tmp_path, "resumed12", 2, bk1)
    assert int(resumed12["count"]) == int(full1["count"]) and np.array_equal(resumed12["step"], full1["step"])
    e = np.abs(resumed12["params"] - full1["params"]).max() / np.abs(full1["params"]).max()
    assert e < 2e-4, e
    for k, v in _hist(resumed12).items():
        np.testing.assert_allclose(v, full1[k][2:], rtol=2e-4, atol=1e-6, err_msg=k)


def test_model_checkpoint_best_only_keeps_the_best_epoch(tmp_path):
    import dib_b200
    x, y = _c0_data(1024)
    xv, yv = _c0_data(256, 1)
    m = _c0_model("fp16", seed=2)
    rec = _recorder()
    best = str(tmp_path / "best.npz")
    every = str(tmp_path / "w{epoch:02d}-{val_loss:.3f}.npz")
    m.fit(x, y, epochs=6, batch_size=128, verbose=False, validation_data=(xv, yv),
          callbacks=[dib_b200.InfoBottleneckAnnealingCallback(1e-1, 1.0, 2, 3),
                     dib_b200.ModelCheckpoint(best, save_best_only=True, save_weights_only=True),
                     dib_b200.ModelCheckpoint(every, save_weights_only=True), rec])
    losses = [logs["val_loss"] for _, logs in rec.logs]
    k = int(np.argmin(losses))
    fresh = _c0_model("fp16", seed=5)
    fresh.load_weights(best)
    assert np.array_equal(fresh.get_flat_weights(), rec.weights[k])
    for e, logs in rec.logs:
        fresh.load_weights(str(tmp_path / f"w{e + 1:02d}-{logs['val_loss']:.3f}.npz"))
        assert np.array_equal(fresh.get_flat_weights(), rec.weights[e])
