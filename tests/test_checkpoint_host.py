"""Host tests of the checkpoint format (dib_b200.checkpoint) and of ModelCheckpoint's bookkeeping: no GPU needed."""
import json
import os

import numpy as np
import pytest

from dib_b200 import checkpoint as C
from dib_b200.keras_compat import BackupAndRestore, ModelCheckpoint


def _synthetic(seed=0, state=False):
    rng = np.random.default_rng(seed)
    shapes = {"feature_encoder_0/dense_0/kernel": (5, 3), "feature_encoder_0/dense_0/bias": (3,),
              "integration_network/dense_0/kernel": (3, 1), "integration_network/dense_0/bias": (1,)}
    arrays = {n: rng.standard_normal(s).astype(np.float32) for n, s in shapes.items()}
    manifest = dict(version=C.FORMAT_VERSION, kind="model" if state else "weights",
                    model={"class": "DistributedIBNet", "config": {"feature_dimensionalities": [5]}},
                    variables=[[n, list(s)] for n, s in shapes.items()])
    if state:
        P = sum(a.size for a in arrays.values())
        manifest["compile"] = {"optimizer": {"class": "Adam", "config": {"learning_rate": 1e-3}}}
        manifest["state"] = {"train_step_count": 7, "beta": 0.5}
        arrays["optimizer/m"] = rng.standard_normal(P).astype(np.float32)
        arrays["optimizer/v"] = rng.random(P).astype(np.float32)
    return manifest, arrays


@pytest.mark.parametrize("state", [False, True])
def test_round_trip(tmp_path, state):
    manifest, arrays = _synthetic(state=state)
    path = tmp_path / "ck.npz"
    C.write(path, manifest, arrays)
    got_manifest, got = C.read(path)
    assert got_manifest == manifest
    assert set(got) == set(arrays)
    for k, a in arrays.items():
        assert got[k].dtype == np.float32 and np.array_equal(got[k], a), k
    # readable without the engine: plain numpy, no pickle
    with np.load(path, allow_pickle=False) as npz:
        assert np.array_equal(npz["integration_network/dense_0/kernel"], arrays["integration_network/dense_0/kernel"])
    names = [n for n, _ in manifest["variables"]]
    shapes = [tuple(s) for _, s in manifest["variables"]]
    flat = C.flatten(got_manifest, got)
    assert flat.size == 5 * 3 + 3 + 3 + 1
    back = C.split(flat, names, shapes)
    assert all(np.array_equal(back[n], arrays[n]) for n in names)
    assert not [f for f in os.listdir(tmp_path) if f != "ck.npz"]           # no temporary file left behind


def test_truncated_file_is_refused(tmp_path):
    manifest, arrays = _synthetic()
    path = tmp_path / "ck.npz"
    C.write(path, manifest, arrays)
    data = path.read_bytes()
    for cut in (len(data) - 1, len(data) // 2, 10, 0):
        path.write_bytes(data[:cut])
        with pytest.raises(ValueError, match="not a readable checkpoint"):
            C.read(path)


def test_every_single_byte_flip_is_refused_or_harmless(tmp_path):
    """A flipped byte in a member's data or header fails its CRC; one in the zip structure fails the zip parser; only bytes
    nothing reads back (timestamps, attributes) may pass -- and then the content read is exactly what was written."""
    manifest, arrays = _synthetic(state=True)
    path = tmp_path / "ck.npz"
    C.write(path, manifest, arrays)
    data = path.read_bytes()
    refused = set()
    for i in range(len(data)):
        bad = bytearray(data)
        bad[i] ^= 0x5A
        path.write_bytes(bytes(bad))
        try:
            m, got = C.read(path)
        except ValueError:
            refused.add(i)
            continue
        assert m == manifest and set(got) == set(arrays), i
        assert all(np.array_equal(got[k], a) for k, a in arrays.items()), i
    payload = [json.dumps(manifest, sort_keys=True).encode()] + [a.tobytes() for a in arrays.values()]
    for blob in payload:
        lo = data.index(blob)
        assert set(range(lo, lo + len(blob))) <= refused
    assert len(refused) > len(data) // 2, (len(refused), len(data))


def test_data_byte_flip_names_crc(tmp_path):
    manifest, arrays = _synthetic()
    path = tmp_path / "ck.npz"
    C.write(path, manifest, arrays)
    data = bytearray(path.read_bytes())
    pos = bytes(data).index(arrays["feature_encoder_0/dense_0/kernel"].tobytes())
    data[pos + 3] ^= 1
    path.write_bytes(bytes(data))
    with pytest.raises(ValueError, match="CRC"):
        C.read(path)


def _write_raw(path, members):
    """An archive written around checkpoint.write's checks: {name: array}, the manifest given as a dict."""
    out = {}
    for k, v in members.items():
        out[k] = (np.frombuffer(json.dumps(v).encode(), dtype=np.uint8) if k == C.MANIFEST else v)
    with open(path, "wb") as fh:
        np.savez(fh, **out)


def test_unknown_version_and_kind_are_refused(tmp_path):
    manifest, arrays = _synthetic()
    for field, value, msg in (("version", 2, "version 2"), ("version", None, "version None"), ("kind", "optimizer", "kind")):
        bad = dict(manifest, **{field: value})
        _write_raw(tmp_path / "ck.npz", dict(arrays, manifest=bad))
        with pytest.raises(ValueError, match=msg):
            C.read(tmp_path / "ck.npz")


def test_renamed_or_reshaped_variable_is_refused(tmp_path):
    manifest, arrays = _synthetic()
    path = tmp_path / "ck.npz"
    # a member whose name or shape disagrees with the manifest
    renamed = dict(arrays)
    renamed["integration_network/dense_0/kernel_"] = renamed.pop("integration_network/dense_0/kernel")
    _write_raw(path, dict(renamed, manifest=manifest))
    with pytest.raises(ValueError, match="'integration_network/dense_0/kernel' has no member"):
        C.read(path)
    reshaped = dict(arrays, **{"feature_encoder_0/dense_0/kernel": np.zeros((3, 5), np.float32)})
    _write_raw(path, dict(reshaped, manifest=manifest))
    with pytest.raises(ValueError, match=r"'feature_encoder_0/dense_0/kernel' is float32 \(3, 5\)"):
        C.read(path)
    wrong_dtype = dict(arrays, **{"feature_encoder_0/dense_0/bias": np.zeros(3, np.float64)})
    _write_raw(path, dict(wrong_dtype, manifest=manifest))
    with pytest.raises(ValueError, match="feature_encoder_0/dense_0/bias"):
        C.read(path)
    # a consistent file checked against a model with a renamed or reshaped variable
    names = [n for n, _ in manifest["variables"]]
    shapes = [tuple(s) for _, s in manifest["variables"]]
    C.check_variables(manifest, names, shapes)
    with pytest.raises(ValueError, match="variable 2 differs.*'integration_network/dense_0/kernel'.*'integration_network/dense_9/kernel'"):
        C.check_variables(manifest, names[:2] + ["integration_network/dense_9/kernel"] + names[3:], shapes)
    with pytest.raises(ValueError, match=r"variable 1 differs.*\(3,\).*\(4,\)"):
        C.check_variables(manifest, names, shapes[:1] + [(4,)] + shapes[2:])
    with pytest.raises(ValueError, match="4 variables.*5.*first unmatched is the model's 'extra'"):
        C.check_variables(manifest, names + ["extra"], shapes + [(1,)])
    with pytest.raises(ValueError, match="4 variables.*3.*first unmatched is the file's 'integration_network/dense_0/bias'"):
        C.check_variables(manifest, names[:3], shapes[:3])


def test_member_that_needs_pickle_is_refused(tmp_path):
    manifest, arrays = _synthetic()
    path = tmp_path / "ck.npz"
    obj = np.empty(2, dtype=object)
    obj[0], obj[1] = {"a": 1}, [2]
    _write_raw(path, dict(arrays, manifest=manifest, extra=obj))
    with pytest.raises(ValueError, match="allow_pickle"):
        C.read(path)
    with pytest.raises(ValueError, match="float32"):
        C.write(path, manifest, dict(arrays, extra=obj))


def test_missing_slots_and_extra_members_are_refused(tmp_path):
    manifest, arrays = _synthetic(state=True)
    path = tmp_path / "ck.npz"
    short = dict(arrays)
    del short["optimizer/v"]
    _write_raw(path, dict(short, manifest=manifest))
    with pytest.raises(ValueError, match="optimizer/v"):
        C.read(path)
    _write_raw(path, dict(arrays, manifest=manifest, stray=np.zeros(1, np.float32)))
    with pytest.raises(ValueError, match="stray"):
        C.read(path)
    weights_manifest, weights = _synthetic()
    _write_raw(path, dict(weights, manifest=dict(weights_manifest, state={})))
    with pytest.raises(ValueError, match="no training state"):
        C.read(path)


def test_failed_write_leaves_previous_file_intact(tmp_path, monkeypatch):
    manifest, arrays = _synthetic(seed=0)
    path = tmp_path / "ck.npz"
    C.write(path, manifest, arrays)
    before = path.read_bytes()
    _, newer = _synthetic(seed=1)

    def crash(src, dst):
        assert os.path.getsize(src) > 0          # the temporary file was written in full
        raise OSError("simulated crash before the rename")

    monkeypatch.setattr(C.os, "replace", crash)
    with pytest.raises(OSError, match="simulated"):
        C.write(path, manifest, newer)
    monkeypatch.undo()
    assert path.read_bytes() == before
    assert os.listdir(tmp_path) == ["ck.npz"]                                 # the temporary file was removed
    _, got = C.read(path)
    assert all(np.array_equal(got[k], arrays[k]) for k in arrays)


# ------------------------------------------------------------------ ModelCheckpoint with a stub model


class _StubModel:
    def __init__(self):
        self.calls = []

    def save(self, path, include_optimizer=True):
        self.calls.append(("save", path))

    def save_weights(self, path):
        self.calls.append(("save_weights", path))


def _drive(cb, logs_per_epoch):
    model = _StubModel()
    cb.set_model(model)
    for epoch, logs in enumerate(logs_per_epoch):
        cb.on_epoch_end(epoch, logs)
    return model.calls


def test_model_checkpoint_formats_epoch_and_logs():
    cb = ModelCheckpoint("run/ep{epoch:03d}-{val_loss:.2f}-{accuracy:.1f}.npz")
    calls = _drive(cb, [dict(val_loss=0.5, accuracy=0.25), dict(val_loss=0.123, accuracy=0.75)])
    assert calls == [("save", "run/ep001-0.50-0.2.npz"), ("save", "run/ep002-0.12-0.8.npz")]
    cb = ModelCheckpoint("w{epoch}.npz", save_weights_only=True)
    assert _drive(cb, [{}, {}, {}]) == [("save_weights", f"w{e}.npz") for e in (1, 2, 3)]


def test_model_checkpoint_best_only_min_max_auto():
    losses = [0.9, 0.7, 0.8, 0.7, 0.6]
    cb = ModelCheckpoint("b{epoch}.npz", save_best_only=True)                           # val_loss, auto -> min
    assert [p for _, p in _drive(cb, [dict(val_loss=v) for v in losses])] == ["b1.npz", "b2.npz", "b5.npz"]
    assert cb.best == 0.6
    accs = [0.5, 0.6, 0.55, 0.6, 0.7]
    for monitor in ("val_accuracy", "accuracy", "val_auc", "pr_auc", "val_precision", "recall"):
        cb = ModelCheckpoint("b{epoch}.npz", monitor=monitor, save_best_only=True)        # auto -> max
        assert [p for _, p in _drive(cb, [{monitor: v} for v in accs])] == ["b1.npz", "b2.npz", "b5.npz"], monitor
    cb = ModelCheckpoint("b{epoch}.npz", monitor="val_accuracy", mode="min", save_best_only=True)
    assert [p for _, p in _drive(cb, [dict(val_accuracy=v) for v in accs])] == ["b1.npz"]
    cb = ModelCheckpoint("b{epoch}.npz", monitor="val_loss", mode="max", save_best_only=True)
    assert [p for _, p in _drive(cb, [dict(val_loss=v) for v in losses])] == ["b1.npz"]
    with pytest.warns(UserWarning, match="fallback to auto"):
        cb = ModelCheckpoint("b{epoch}.npz", mode="sideways", save_best_only=True)
    assert [p for _, p in _drive(cb, [dict(val_loss=v) for v in losses])] == ["b1.npz", "b2.npz", "b5.npz"]


def test_model_checkpoint_initial_value_threshold_and_missing_monitor():
    cb = ModelCheckpoint("b{epoch}.npz", save_best_only=True, initial_value_threshold=0.75)
    assert [p for _, p in _drive(cb, [dict(val_loss=v) for v in (0.9, 0.8, 0.7, 0.75)])] == ["b3.npz"]
    cb = ModelCheckpoint("b{epoch}.npz", monitor="val_auc", save_best_only=True, initial_value_threshold=0.9)
    assert [p for _, p in _drive(cb, [dict(val_auc=v) for v in (0.8, 0.9, 0.95)])] == ["b3.npz"]
    cb = ModelCheckpoint("b{epoch}.npz", save_best_only=True)
    with pytest.warns(UserWarning, match="val_loss available, skipping"):
        assert _drive(cb, [dict(loss=0.3)]) == []
    cb = ModelCheckpoint("b{epoch}.npz")                  # without save_best_only every epoch is saved, monitor or not
    assert len(_drive(cb, [dict(loss=0.3)] * 2)) == 2


def test_checkpoint_callbacks_refuse_batch_frequencies():
    with pytest.raises(ValueError, match="every so many batches is not implemented"):
        ModelCheckpoint("x.npz", save_freq=100)
    with pytest.raises(ValueError, match="Unrecognized save_freq"):
        ModelCheckpoint("x.npz", save_freq="batch")
    with pytest.raises(ValueError, match="epoch ends"):
        BackupAndRestore("dir", save_freq=10)


def test_callbacks_namespace():
    import dib_b200
    assert dib_b200.callbacks.ModelCheckpoint is ModelCheckpoint
    assert dib_b200.callbacks.BackupAndRestore is BackupAndRestore
    assert dib_b200.callbacks.Callback is dib_b200.Callback


def test_metric_configs_round_trip():
    from dib_b200 import metrics as M
    objs = [M.AUC(num_thresholds=57, curve="PR", summation_method="minoring", from_logits=True, name="pr"),
            M.Precision(0.7), M.Recall(thresholds=0.3, name="r"), M.BinaryAccuracy(threshold=0.2),
            M.BinaryCrossentropy(from_logits=True, name="bce"), M.SparseCategoricalCrossentropy(from_logits=True),
            M.SparseCategoricalAccuracy(name="accuracy"), M.MeanSquaredError(name="mse"), M.MeanAbsoluteError()]
    for m in objs:
        spec = json.loads(json.dumps(M.serialize(m)))
        back = M.deserialize(spec)
        assert type(back) is type(m) and back.get_config() == m.get_config(), m
        assert vars(back) == vars(m), m
    assert M.deserialize("accuracy") == "accuracy"
    with pytest.raises(ValueError, match="unknown metric"):
        M.deserialize({"class": "Callback", "config": {}})
