"""Cost of compiled metrics in the training step: ``train_on_batch`` under CUDA-graph replay without metrics, with mean
metrics, and with confusion-matrix metrics, alternated in one session so that every mode sees the same card state.

Shapes (fp16): C0 (bench.py: 16 scalar features, PE, enc [128, 128], int [256, 256] -> 1, batch 65 536) and the nb-radial
shape (100 features, tanh, no PE, int [256, 256, 256] -> 1, batch 256).  x, y and the sample weights live on the device.
Modes, on the logit model compiled with BinaryCrossentropy(from_logits=True):
  none  metrics=['accuracy'] (the parent's step)
  mean  + 'mse', 'mae', BinaryCrossentropy(from_logits=True), weighted 'binary_accuracy'
  auc   + AUC(from_logits=True) (200 thresholds)
and, since Precision / Recall need probabilities, on the same shape with output_activation_fn='sigmoid' and
BinaryCrossentropy(from_logits=False):
  probs_none  metrics=['accuracy']
  probs_conf  + AUC(), Precision(), Recall()
For every (shape, mode) it prints one JSON line with the median and the spread (min, max) of ms per step over ``--rounds``
rounds of ``--steps`` steps (CUDA events around each round); the first line names the GPU, its power limit and SM clock.

    python tools/bench_metrics.py [--steps 20] [--rounds 7] [--warmup 3] [--out F]
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


def modes():
    from dib_b200 import metrics as M
    return {
        "none": (False, ["accuracy"], None),
        "mean": (False, ["accuracy", "mse", "mae", M.BinaryCrossentropy(from_logits=True)], ["binary_accuracy"]),
        "auc": (False, ["accuracy", M.AUC(from_logits=True)], None),
        "probs_none": (True, ["accuracy"], None),
        "probs_conf": (True, ["accuracy", M.AUC(), M.Precision(), M.Recall()], None),
    }


def make(shape, probs, metrics, weighted):
    import dib_b200
    s = SHAPES[shape]
    m = dib_b200.DistributedIBNet(s["fdims"], [128, 128], s["integ"], 1, use_positional_encoding=s["pe"], activation_fn=s["act"],
                                  feature_embedding_dimension=32, precision="fp16", seed=0,
                                  output_activation_fn="sigmoid" if probs else None)
    m.compile(optimizer=dib_b200.Adam(3e-4), loss=dib_b200.losses.BinaryCrossentropy(from_logits=not probs), metrics=metrics,
              weighted_metrics=weighted)
    m.beta.assign(1e-3)
    return m


def bench(shape, steps, rounds, warmup):
    s = SHAPES[shape]
    B, D = s["batch"], sum(s["fdims"])
    rng = np.random.default_rng(0)
    xh = rng.standard_normal((B, D)).astype(np.float32)
    x = torch.from_numpy(xh).cuda()
    y = torch.from_numpy((xh[:, :1] * xh[:, 1:2] > 0).astype(np.float32)).cuda()
    w = torch.from_numpy(rng.uniform(0, 5, B).astype(np.float32)).cuda()
    models = {name: make(shape, *spec) for name, spec in modes().items()}
    names = list(models)
    for name in names:                                  # two eager steps per graph key, then capture and replay
        for _ in range(max(warmup, 3)):
            models[name].train_on_batch(x, y, sample_weight=w, sync=False)
    torch.cuda.synchronize()
    times = {name: [] for name in names}
    for r in range(rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            m = models[name]
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                m.train_on_batch(x, y, sample_weight=w, sync=False)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / steps)
    out = []
    for name in names:
        assert len(models[name]._graphs) == 1, list(models[name]._graphs)       # replayed, not eager
        t = np.asarray(times[name])
        out.append(dict(shape=shape, precision="fp16", batch=B, mode=name, tail_floats=models[name]._tail_len,
                        ms_per_step_median=round(float(np.median(t)), 4), ms_per_step_min=round(float(t.min()), 4),
                        ms_per_step_max=round(float(t.max()), 4), rounds=rounds, steps_per_round=steps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics needs a CUDA device")
    lines = [gpu_info()]
    print(json.dumps(lines[0]), flush=True)
    for shape in SHAPES:
        for rec in bench(shape, a.steps, a.rounds, a.warmup):
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
