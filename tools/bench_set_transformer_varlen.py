"""Time SetTransformerIBNet's training step on sets of different sizes (variable_set_sizes=True) at nb-particle cell 8's network
(12 features -> PE 5 -> [128, 128] -> E 32, 6 blocks of 12 heads x 128, FF [128, 32], head [256] -> 1, BCE on logits):

  (a) every set of 50 particles on the variable-size path (Lmax = 50), and the fixed-size model at L = 50 in the same run;
  (b) sizes uniform in [30, 100], Lmax = 100;
  (c) sizes uniform in [30, 256], Lmax = 256.

For every (case, batch of sets) it prints one JSON line: ms per step (median of CUDA-event intervals between consecutive
graph-replayed steps; the size vector changes every step for (b) and (c)), the attention kernels' share of one profiled eager
step (dib_profile_* ranges st_attn_fwd_b* + st_attn_bwd_b* over the sum of all ranges), and the workspace bytes.  The first
line names the GPU, its power limit and its maximum SM clock.

    python tools/bench_set_transformer_varlen.py [--batches 32,256,1024] [--cases a,b,c] [--steps 20] [--warmup 3] [--out F]
"""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infonce import gpu_info, profile_split  # noqa: E402
from bench_set_transformer import timed  # noqa: E402

D, E, H, DK, BLOCKS = 12, 32, 12, 128, 6
CASES = {"a": (50, 50, 50), "b": (100, 30, 100), "c": (256, 30, 256)}     # Lmax, smallest and largest size


def make(Lmax, variable, precision):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(D, [128, 128], E, Lmax, key_dim=DK, number_heads=H, number_attention_blocks=BLOCKS,
                                     precision=precision, seed=0, variable_set_sizes=variable)
    m.compile(optimizer=dib_b200.Adam(1e-4), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
    m.beta.assign(1e-3)
    return m


def bench(case, B, steps, warmup, precision, variable=True):
    Lmax, lo, hi = CASES[case]
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((B, Lmax, D)).astype(np.float32)).cuda()
    y = torch.from_numpy((rng.random((B, 1)) > 0.5).astype(np.float32)).cuda()
    sizes = [torch.from_numpy(rng.integers(lo, hi + 1, B).astype(np.int32)).cuda() for _ in range(8)]
    m = make(Lmax, variable, precision)
    k = {"i": 0}

    def step():
        k["i"] += 1
        if variable:
            m.train_on_batch((x, sizes[k["i"] % len(sizes)]), y, sync=False)
        else:
            m.train_on_batch(x, y, sync=False)
    dts = timed(step, steps, warmup)
    prof = profile_split(m, (x, sizes[0]) if variable else x, y)
    attn = sum(t for lab, t in prof.items() if lab.startswith("st_attn_"))
    total = sum(prof.values())
    res = {"case": case, "path": "variable" if variable else "fixed", "precision": precision, "batch_sets": B, "Lmax": Lmax,
           "sizes": [lo, hi], "mean_size": round(float(torch.stack(sizes).float().mean()), 2) if variable else Lmax,
           "steps": steps, "ms_per_step_median": round(float(np.median(dts)), 4), "ms_per_step_min": round(float(np.min(dts)), 4),
           "graph_replay": bool(m._graphs), "attention_share_of_profiled_step": round(attn / total, 4) if total else None,
           "attention_ms_profiled": round(attn, 4), "profiled_step_ms": round(total, 4),
           "workspace_bytes": int(m._lib.dib_workspace_bytes(m._handle)), "kernel_info": m.kernel_info(B)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,256,1024")
    ap.add_argument("--cases", default="a,b,c")
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_set_transformer_varlen.py needs a CUDA device (H100)")
    lines = [json.dumps(gpu_info())]
    print(lines[-1], flush=True)
    for case in a.cases.split(","):
        for B in [int(b) for b in a.batches.split(",")]:
            runs = [(case, True)] + ([(case, False)] if case == "a" else [])    # (a): the fixed-size model alongside
            for c, variable in runs:
                lines.append(json.dumps(bench(c, B, a.steps, a.warmup, a.precision, variable)))
                print(lines[-1], flush=True)
                gc.collect()                     # the model and its captured graphs reference each other
                torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
