"""Time one rank of data-parallel InfoNCE training with global negatives (losses.InfoNCE(..., negatives='global'), DESIGN.md
section 7) on one GPU: a virtual rank that owns n_global / N rows of the double-pendulum shape (as tools/bench_infonce.py:
features [2, 1, 2, 1], encoders [128, 128], integration [256, 256], InfoNCE dimension 64, output encoder 6 -> PE 30 ->
[128, 128] -> 64, similarity 'l2', temperature 1).

The rank's step is four CUDA graphs -- phase 1 (forward, output encoder, its rows of e_all), phase 2 (row / column
log-sum-exps of its rows against all n_global rows, stats), phase 3 (gradient sweeps and backward), the optimizer -- with
the two all-gathers and the all-reduce between them.  Those collectives are not run here (one process); what they would
move is computed from the shapes.  Each timed phase is the median over the steps of CUDA-event intervals around its graph
replay.  The other ranks' rows of e_all are real embeddings (phase 1 run once per row block before timing).

For every (precision, n_global, N) it prints one JSON line; the first line names the GPU, its power limit and its maximum
SM clock.

    python tools/bench_infonce_dp.py [--globals 8192,65536] [--ranks 1,2,4,8] [--precisions fp16,fp32] [--steps 10]
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

from bench_infonce import gpu_info, make  # noqa: E402


def collective_bytes(m, n_global, N):
    """Bytes each collective leaves on every rank (its output) and each rank contributes, from the shapes."""
    d, n = m.output_dimensionality, n_global // N
    stats = m._P + m.number_features + 3
    return {"all_gather_e_all": {"out_bytes": 4 * n_global * 2 * d, "per_rank_in_bytes": 4 * n * 2 * d},
            "all_gather_lse_all": {"out_bytes": 4 * n_global * 2, "per_rank_in_bytes": 4 * n * 2},
            "all_reduce_grads_stats": {"bytes": 4 * stats}}


def bench(precision, n_global, N, steps, warmup):
    m = make(precision)
    n = n_global // N
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((n_global, 6)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.standard_normal((n_global, 6)).astype(np.float32)).cuda()
    m._ensure_handle(n)
    m._set_device_step(False)
    e_all, lse_all = m._infonce_buffers(n_global)
    for r in reversed(range(N)):          # every row block of e_all; block 0 (this rank's) last, so the workspace is its
        sl = slice(r * n, (r + 1) * n)
        m._infonce_forward(x[sl], y[sl], e_all, n_global, r * n, None, 0, r * n, training=True)
    m._infonce_lse(n, e_all, lse_all, n_global, 0, m._gradstats[m._P:])
    lse_all.copy_(lse_all[:n].repeat(N, 1)[:n_global])   # the other ranks' (r, c) rows: plausible values
    xs, ys = x[:n].contiguous(), y[:n].contiguous()
    phases = {
        "phase1_forward": lambda: m._infonce_forward(xs, ys, e_all, n_global, 0, None, 0, 0, training=True),
        "phase2_lse": lambda: m._infonce_lse(n, e_all, lse_all, n_global, 0, m._gradstats[m._P:]),
        "phase3_backward": lambda: m._infonce_backward(xs, e_all, lse_all, n_global, 0, None, 0, 0),
        "optimizer": m._adam,
    }
    graphs = {}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):          # one eager pass per phase before capture (lazy kernel attribute set-up)
        for fn in phases.values():
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for name, fn in phases.items():
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        graphs[name] = g
    times = {k: [] for k in phases}
    total = []
    for it in range(warmup + steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(graphs) + 1)]
        ev[0].record()
        for i, g in enumerate(graphs.values()):
            g.replay()
            ev[i + 1].record()
        torch.cuda.synchronize()
        if it >= warmup:
            for i, k in enumerate(graphs):
                times[k].append(ev[i].elapsed_time(ev[i + 1]))
            total.append(ev[0].elapsed_time(ev[-1]))
    res = {"precision": precision, "n_global": n_global, "ranks": N, "rows_per_rank": n, "steps": steps,
           "ms_median": {k: round(float(np.median(v)), 4) for k, v in times.items()},
           "ms_total_median": round(float(np.median(total)), 4),
           "collectives": collective_bytes(m, n_global, N), "kernel_info": m.kernel_info(n)}
    del graphs, m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--globals", default="8192,65536")
    ap.add_argument("--ranks", default="1,2,4,8")
    ap.add_argument("--precisions", default="fp16,fp32")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infonce_dp.py needs a CUDA device (H100)")
    lines = [json.dumps(gpu_info())]
    print(lines[-1], flush=True)
    for prec in a.precisions.split(","):
        for ng in [int(b) for b in a.globals.split(",")]:
            for N in [int(r) for r in a.ranks.split(",")]:
                if ng % N:
                    raise SystemExit(f"n_global {ng} does not split into {N} equal shards")
                lines.append(json.dumps(bench(prec, ng, N, a.steps, a.warmup)))
                print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
