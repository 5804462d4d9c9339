"""Time the InfoNCE training step (losses.InfoNCE: output encoder + streaming InfoNCE kernels) on the double-pendulum
shape of train.py:116-126: features [2, 1, 2, 1], encoders [128, 128], integration [256, 256], InfoNCE dimension 64,
output encoder 6 -> PE 30 -> [128, 128] -> 64, similarity 'l2', temperature 1.

For every (precision, batch) it prints one JSON line: ms per step (median of CUDA-event intervals between consecutive
graph-replayed steps), the dib_profile_* launch-group split of one eager step, and the workspace bytes.  The first line
names the GPU, its power limit and its maximum SM clock.

    python tools/bench_infonce.py [--batches 128,2048,8192,65536] [--precisions fp32,fp16] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": repr(e)}


def make(precision):
    import dib_b200
    m = dib_b200.DistributedIBNet([2, 1, 2, 1], [128, 128], [256, 256], 64, output_activation_fn=None, precision=precision,
                                  seed=0)
    m.compile(optimizer=dib_b200.Adam(1e-4), loss=dib_b200.losses.InfoNCE(6, [128, 128], similarity="l2", temperature=1.0))
    m.beta.assign(1e-3)
    return m


def profile_split(m, x, y):
    lib = m._lib
    lib.dib_profile_enable(m._handle, 1)
    m.compute_gradients(x, y)
    torch.cuda.synchronize()
    cap = 512
    ms = (ctypes.c_float * cap)()
    labels = ctypes.create_string_buffer(1 << 16)
    k = lib.dib_profile_read(m._handle, labels, len(labels), ms, cap)
    lib.dib_profile_enable(m._handle, 0)
    split = {}
    for lab, t in zip(labels.value.decode().split("\n")[:k], ms[:k]):
        split[lab] = round(split.get(lab, 0.0) + float(t), 4)
    return split


def bench(precision, B, steps, warmup):
    m = make(precision)
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((B, 6)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.standard_normal((B, 6)).astype(np.float32)).cuda()
    for _ in range(max(warmup, 3)):                      # two eager steps, then capture and replay
        m.train_on_batch(x, y, sync=False)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for i in range(steps):
        m.train_on_batch(x, y, sync=False)
        ev[i + 1].record()
    torch.cuda.synchronize()
    dts = [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
    res = {"precision": precision, "batch": B, "steps": steps, "ms_per_step_median": round(float(np.median(dts)), 4),
           "ms_per_step_min": round(float(np.min(dts)), 4), "graph_replay": bool(m._graphs),
           "workspace_bytes": int(m._lib.dib_workspace_bytes(m._handle)), "kernel_info": m.kernel_info(B)}
    res["profile_ms"] = profile_split(m, x, y)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,2048,8192,65536")
    ap.add_argument("--precisions", default="fp32,fp16")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infonce.py needs a CUDA device (H100)")
    lines = [json.dumps(gpu_info())]
    print(lines[-1], flush=True)
    for prec in a.precisions.split(","):
        for B in [int(b) for b in a.batches.split(",")]:
            lines.append(json.dumps(bench(prec, B, a.steps, a.warmup)))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
