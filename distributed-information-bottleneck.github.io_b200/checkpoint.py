"""Checkpoint files: ``model.save_weights`` / ``model.save`` write one file, ``model.load_weights`` /
``models.load_model`` read it back (``callbacks.ModelCheckpoint`` and ``callbacks.BackupAndRestore`` drive them from
``fit``).

A checkpoint is a NumPy ``.npz`` archive (a zip of ``.npy`` members, each CRC-checked), written without pickle and read with
``allow_pickle=False``.  The member ``manifest`` holds UTF-8 JSON:

    version     FORMAT_VERSION
    kind        'weights' (save_weights) or 'model' (save)
    model       {"class": class name, "config": constructor arguments}
    variables   [[name, shape], ...] in the model's flat order
    compile     ('model' files saved with include_optimizer) optimizer with its learning rate, loss, compiled metrics
    state       (the same files) beta, optimizer step, Philox step count, noise and shuffle seeds, inference calls,
                completed epochs

Every variable is its own float32 member under its name, in Keras orientation (a Dense kernel is [in, out]), so the file
reads without the engine: ``np.load(path)["integration_network/dense_0/kernel"]``.  A file with a state also holds the two
optimizer slot buffers as flat float32 members ``optimizer/m`` and ``optimizer/v`` (Adam m / v, SGD velocity, RMSprop mean
square / momentum) in the same flat order.

This module needs only numpy, json and os: the format is tested without a GPU."""
from __future__ import annotations

import json
import os
import tempfile
import zipfile

import numpy as np

FORMAT_VERSION = 1
KINDS = ("weights", "model")
MANIFEST = "manifest"
SLOTS = ("optimizer/m", "optimizer/v")


def write(path, manifest, arrays):
    """Write ``manifest`` (a JSON-able dict) and ``arrays`` ({member name: float32 array}) to ``path`` atomically: into a
    temporary file in the same directory, flushed and fsync'ed, then renamed over ``path``.  A crash or an error before the
    rename leaves a previous file at ``path`` as it was."""
    path = os.fspath(path)
    if MANIFEST in arrays:
        raise ValueError(f"{MANIFEST!r} is reserved for the manifest")
    members = {MANIFEST: np.frombuffer(json.dumps(manifest, sort_keys=True).encode("utf-8"), dtype=np.uint8)}
    for name, a in arrays.items():
        a = np.asarray(a)
        if a.dtype != np.float32:
            raise ValueError(f"member {name!r} is {a.dtype}; checkpoint members are float32")
        members[name] = a
    directory = os.path.dirname(os.path.abspath(path))
    fd, tmp = tempfile.mkstemp(prefix="." + os.path.basename(path) + ".", suffix=".tmp", dir=directory)
    try:
        with os.fdopen(fd, "wb") as fh:
            np.savez(fh, **members)
            fh.flush()
            os.fsync(fh.fileno())
        os.replace(tmp, path)
    except BaseException:
        try:
            os.remove(tmp)
        except OSError:
            pass
        raise
    try:                                  # make the rename itself durable
        dfd = os.open(directory, os.O_RDONLY)
    except OSError:
        return
    try:
        os.fsync(dfd)
    except OSError:
        pass
    finally:
        os.close(dfd)


def read(path):
    """(manifest, {member name: array}) of the checkpoint at ``path``.  Raises ValueError, before returning anything, on a
    file that is not a complete, uncorrupted checkpoint of a known version: a truncated or altered archive (zip structure or
    member CRC), a member that needs pickle, a manifest without the fields of its kind, or a variable missing, misnamed,
    misshaped or not float32 (the first such variable is named)."""
    path = os.fspath(path)
    try:
        with zipfile.ZipFile(path) as zf:
            bad = zf.testzip()                         # reads every member and checks its CRC-32
        if bad is not None:
            raise ValueError(f"member {bad!r} fails its CRC check")
        with np.load(path, allow_pickle=False) as npz:
            members = {name: npz[name] for name in npz.files}
    except ValueError as e:
        raise ValueError(f"{path}: not a readable checkpoint: {e}") from e
    except Exception as e:                             # zipfile.BadZipFile, zlib / struct errors, EOFError, OSError
        raise ValueError(f"{path}: not a readable checkpoint (truncated or corrupted): {e!r}") from e
    if MANIFEST not in members:
        raise ValueError(f"{path}: no {MANIFEST!r} member: not a checkpoint")
    raw = members.pop(MANIFEST)
    try:
        if raw.dtype != np.uint8 or raw.ndim != 1:
            raise ValueError(f"the manifest member is {raw.dtype} {raw.shape}")
        manifest = json.loads(raw.tobytes().decode("utf-8"))
        if not isinstance(manifest, dict):
            raise ValueError("the manifest is not a JSON object")
    except (ValueError, UnicodeDecodeError) as e:
        raise ValueError(f"{path}: unreadable manifest: {e}") from e
    version = manifest.get("version")
    if version != FORMAT_VERSION:
        raise ValueError(f"{path}: checkpoint format version {version!r}; this engine reads version {FORMAT_VERSION}")
    kind = manifest.get("kind")
    if kind not in KINDS:
        raise ValueError(f"{path}: unknown checkpoint kind {kind!r} (expected one of {KINDS})")
    if kind == "weights" and ("state" in manifest or "compile" in manifest):
        raise ValueError(f"{path}: a 'weights' checkpoint carries no training state")
    for field in ("model", "variables") + (("compile",) if "state" in manifest else ()):
        if field not in manifest:
            raise ValueError(f"{path}: the manifest has no {field!r} field")
    variables = manifest["variables"]
    if not isinstance(variables, list):
        raise ValueError(f"{path}: the manifest's variable list is not a list")
    expected = set()
    for k, entry in enumerate(variables):
        if not (isinstance(entry, list) and len(entry) == 2 and isinstance(entry[0], str) and isinstance(entry[1], list)
                and all(isinstance(d, int) and d >= 0 for d in entry[1])):
            raise ValueError(f"{path}: variable entry {k} is not [name, shape]: {entry!r}")
        name, shape = entry[0], tuple(entry[1])
        a = members.get(name)
        if a is None:
            raise ValueError(f"{path}: variable {k} {name!r} has no member")
        if a.dtype != np.float32 or a.shape != shape:
            raise ValueError(f"{path}: variable {k} {name!r} is {a.dtype} {a.shape}; the manifest says float32 {shape}")
        expected.add(name)
    if "state" in manifest:
        P = sum(int(np.prod(s)) for _, s in variables)
        for name in SLOTS:
            a = members.get(name)
            if a is None or a.dtype != np.float32 or a.shape != (P,):
                raise ValueError(f"{path}: optimizer slot {name!r} is missing or not float32 ({P},)")
            expected.add(name)
    extra = sorted(set(members) - expected)
    if extra:
        raise ValueError(f"{path}: members the manifest does not list: {extra[:3]}")
    return manifest, members


def check_variables(manifest, names, shapes, what="the model"):
    """Raise ValueError naming the first variable where the file's [(name, shape)] differs from ``names`` / ``shapes`` (the
    receiving model's, in flat order)."""
    file_vars = [(n, tuple(s)) for n, s in manifest["variables"]]
    want = [(n, tuple(s)) for n, s in zip(names, shapes)]
    for k, (a, b) in enumerate(zip(file_vars, want)):
        if a != b:
            raise ValueError(f"variable {k} differs: the file has {a[0]!r} {a[1]}, {what} has {b[0]!r} {b[1]}")
    if len(file_vars) != len(want):
        k = min(len(file_vars), len(want))
        first = (f"the file's {file_vars[k][0]!r}" if len(file_vars) > k else f"{what}'s {want[k][0]!r}")
        raise ValueError(f"the file has {len(file_vars)} variables, {what} has {len(want)}: first unmatched is {first}")


def flatten(manifest, members):
    """The file's variables concatenated in flat order (float32 [P])."""
    parts = [members[name].reshape(-1) for name, _ in manifest["variables"]]
    return np.concatenate(parts) if parts else np.zeros(0, np.float32)


def split(flat, names, shapes):
    """{name: array of shape} cut from the flat float32 vector, in order."""
    out, off = {}, 0
    for name, shape in zip(names, shapes):
        size = int(np.prod(shape))
        out[name] = np.ascontiguousarray(flat[off:off + size]).reshape(shape)
        off += size
    if off != flat.size:
        raise ValueError(f"{flat.size} values for variables of {off} values")
    return out
