"""Cost of per-sample weights in the training step: unweighted, ``sample_weight=`` and ``class_weight=`` steps of
``train_on_batch`` under CUDA-graph replay, alternated in one session so that all three see the same card state.

Shapes: C0 (bench.py: 16 scalar features, PE, enc [128, 128], int [256, 256] -> 1, BCE on logits, batch 65 536) in fp16 and
bf16, and the nb-radial shape (C4: 100 features, tanh, no PE, int [256, 256, 256], batch 256) in fp16.  x and y live on the
device; the weights are a host float32 array per step (sample_weight: checked on the host, one 4 n-byte copy) or the class
table {0: 1, 1: 20} (class_weight: the labels read back for the range check, the rows mapped on the device).

For every (shape, precision, mode) it prints one JSON line with the median and the spread (min, max) of ms per step over
``--rounds`` rounds of ``--steps`` steps (CUDA events around each round); the first line names the GPU, its power limit and
its maximum SM clock.

    python tools/bench_sample_weights.py [--steps 20] [--rounds 7] [--warmup 3] [--out F]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infonce import gpu_info  # noqa: E402

SHAPES = {
    "C0": dict(fdims=[1] * 16, integ=[256, 256], act="relu", pe=True, batch=65536),
    "nb-radial": dict(fdims=[1] * 100, integ=[256, 256, 256], act="tanh", pe=False, batch=256),
}
CLASS_WEIGHT = {0: 1.0, 1: 20.0}


def make(shape, precision):
    import dib_b200
    s = SHAPES[shape]
    m = dib_b200.DistributedIBNet(s["fdims"], [128, 128], s["integ"], 1, use_positional_encoding=s["pe"], activation_fn=s["act"],
                                  feature_embedding_dimension=32, precision=precision, seed=0)
    m.compile(optimizer=dib_b200.Adam(3e-4), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
    m.beta.assign(1e-3)
    return m


def bench(shape, precision, steps, rounds, warmup):
    s = SHAPES[shape]
    B, D = s["batch"], sum(s["fdims"])
    rng = np.random.default_rng(0)
    xh = rng.standard_normal((B, D)).astype(np.float32)
    x = torch.from_numpy(xh).cuda()
    y = torch.from_numpy((xh[:, :1] * xh[:, 1:2] > 0).astype(np.float32)).cuda()
    ws = [rng.uniform(0, 5, B).astype(np.float32) for _ in range(4)]
    m = make(shape, precision)
    k = {"i": 0}

    def step(mode):
        k["i"] += 1
        if mode == "unweighted":
            m.train_on_batch(x, y, sync=False)
        elif mode == "sample_weight":
            m.train_on_batch(x, y, sample_weight=ws[k["i"] % len(ws)], sync=False)
        else:
            m.train_on_batch(x, y, class_weight=CLASS_WEIGHT, sync=False)
    modes = ["unweighted", "sample_weight", "class_weight"]
    for mode in modes:                                  # two eager steps per graph key, then capture and replay
        for _ in range(max(warmup, 3)):
            step(mode)
    torch.cuda.synchronize()
    times = {mode: [] for mode in modes}
    for r in range(rounds):
        for mode in (modes if r % 2 == 0 else modes[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                step(mode)
            b.record()
            torch.cuda.synchronize()
            times[mode].append(a.elapsed_time(b) / steps)
    assert sorted(k[-1] for k in m._graphs) == [False, True], list(m._graphs)   # one unweighted, one weighted graph
    out = []
    for mode in modes:
        t = np.asarray(times[mode])
        out.append(dict(shape=shape, precision=precision, batch=B, mode=mode, ms_per_step_median=round(float(np.median(t)), 4),
                        ms_per_step_min=round(float(t.min()), 4), ms_per_step_max=round(float(t.max()), 4),
                        rounds=rounds, steps_per_round=steps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_weights needs a CUDA device")
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    for shape, prec in (("C0", "fp16"), ("C0", "bf16"), ("nb-radial", "fp16")):
        for rec in bench(shape, prec, a.steps, a.rounds, a.warmup):
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
