"""Cost of checkpoints: one ``model.save`` (the full training state) and one ``model.save_weights``, and one ``fit`` epoch with
and without ``BackupAndRestore`` (a full-state save at every epoch end), at two shapes.

Shapes (fp16, as bench.py runs them): C0 (16 scalar features, PE, enc [128, 128], int [256, 256] -> 1, batch 65 536, an epoch
of 8 steps) and nb-radial (100 features, tanh, no PE, int [256, 256, 256], batch 256, an epoch of 52 steps as in the
notebook).  Saves go to a temporary directory; their times are host-clock times of the whole call (device-to-host copy of
the state, zip writing, fsync, rename).  The fit modes are alternated in one session; each round times ``--epochs`` epochs
of one ``fit`` call after a warm-up fit that captured the step's CUDA graphs.

One JSON line per measurement with the median and the spread (min, max) over ``--rounds`` rounds; the first line names the
GPU, its power limit and its maximum SM clock.

    python tools/bench_checkpoint.py [--rounds 5] [--epochs 3] [--out F]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infonce import gpu_info  # noqa: E402

SHAPES = {
    "C0": dict(fdims=[1] * 16, integ=[256, 256], act="relu", pe=True, batch=65536, steps=8),
    "nb-radial": dict(fdims=[1] * 100, integ=[256, 256, 256], act="tanh", pe=False, batch=256, steps=52),
}


def make(shape):
    import dib_b200
    s = SHAPES[shape]
    m = dib_b200.DistributedIBNet(s["fdims"], [128, 128], s["integ"], 1, use_positional_encoding=s["pe"], activation_fn=s["act"],
                                  feature_embedding_dimension=32, precision="fp16", seed=0)
    m.compile(optimizer=dib_b200.Adam(3e-4), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
    m.beta.assign(1e-3)
    return m


def _stats(t):
    t = np.asarray(t) * 1e3
    return dict(ms_median=round(float(np.median(t)), 3), ms_min=round(float(t.min()), 3), ms_max=round(float(t.max()), 3))


def bench(shape, rounds, epochs, tmp):
    import dib_b200
    s = SHAPES[shape]
    B, D = s["batch"], sum(s["fdims"])
    N = B * s["steps"]
    rng = np.random.default_rng(0)
    xh = rng.standard_normal((N, D)).astype(np.float32)
    x = torch.from_numpy(xh).cuda()
    y = torch.from_numpy((xh[:, :1] * xh[:, 1:2] > 0).astype(np.float32)).cuda()
    m = make(shape)
    backup = os.path.join(tmp, f"backup_{shape}")
    fit = lambda n, cbs: m.fit(x, y, batch_size=B, epochs=n, verbose=False, shuffle=True, callbacks=cbs)
    fit(2, [])
    fit(2, [dib_b200.BackupAndRestore(backup)])
    torch.cuda.synchronize()
    path = os.path.join(tmp, f"{shape}.npz")
    m.save(path)
    state_bytes = os.path.getsize(path)
    times = {k: [] for k in ("save", "save_weights", "epoch", "epoch_backup")}
    for r in range(rounds):
        t0 = time.perf_counter()
        m.save(path)
        times["save"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        m.save_weights(path)
        times["save_weights"].append(time.perf_counter() - t0)
        for mode in (("epoch", "epoch_backup") if r % 2 == 0 else ("epoch_backup", "epoch")):
            cbs = [dib_b200.BackupAndRestore(backup)] if mode == "epoch_backup" else []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fit(epochs, cbs)
            torch.cuda.synchronize()
            times[mode].append((time.perf_counter() - t0) / epochs)
    base = dict(shape=shape, precision="fp16", params=m.count_params(), state_file_bytes=state_bytes, batch=B,
                steps_per_epoch=s["steps"], rounds=rounds)
    return [dict(base, what=k, **_stats(v)) for k, v in times.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpoint needs a CUDA device")
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for shape in SHAPES:
            for rec in bench(shape, a.rounds, a.epochs, tmp):
                print(json.dumps(rec), flush=True)
                lines.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
