"""Per-probe information map timings: the card, dib_mi_bounds_at_probes at nb-particle's shape (one particle type: 10 000
probes, 16 batches x 25 600 rows, E = 32), estimate_mi_bounds_at_probes end to end through the notebook network, and the
float64 numpy oracle on a slice as the CPU baseline.  One JSON line per row.

    python tools/bench_probe_information.py [--out F]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_FP64_TENSOR = 67e12          # H100 SXM data sheet, FP64 tensor core, dense


def emit(out, row):
    line = json.dumps(row)
    print(line, flush=True)
    if out:
        with open(out, "a") as fh:
            fh.write(line + "\n")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")]
    return dict(row="card", name=name, power_limit=power, max_sm_clock=clock)


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    out = ap.parse_args().out
    import dib_b200
    from dib_b200 import utils
    from tests import probe_information_oracle as PO
    assert torch.cuda.is_available(), "this benchmark needs the GPU"
    emit(out, card())
    rng = np.random.default_rng(0)
    E, M, B, N = 32, 10000, 16, 25600
    P = torch.from_numpy(np.concatenate([rng.standard_normal((M, E)), rng.uniform(-4, -2, (M, E))], 1).astype(np.float32)).cuda()
    D = torch.from_numpy(np.concatenate([rng.standard_normal((B * N, E)), rng.uniform(-4, -2, (B * N, E))], 1)
                         .astype(np.float32)).cuda()
    off = torch.arange(B + 1, dtype=torch.int64, device="cuda") * N
    ms = time_ms(lambda: utils.mi_bounds_at_probes(P, D, off, None, 1), 5)
    pairs = M * B * N
    flops = pairs * 2 * (2 * E + 1)                       # the expanded quadratic form, one multiply-add per K term
    emit(out, dict(row="kernel", shape=f"M={M} B={B} N={N} E={E}", ms_per_map=round(ms, 3), pairs_per_s=pairs / ms * 1e3,
                    fp64_mma_flops=flops, share_of_datasheet_fp64_tensor_67tflops=flops / (ms * 1e-3) / DATASHEET_FP64_TENSOR))
    m = dib_b200.SetTransformerIBNet(12, [256, 256], 32, 50, key_dim=128, number_heads=12, number_attention_blocks=6)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True))
    m._ensure_handle(32)                                   # a model trained at batch 32
    x = rng.standard_normal((2000, 50, 12)).astype(np.float32)
    probes = rng.standard_normal((M, 12)).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    ms_e2e = time_ms(lambda: utils.estimate_mi_bounds_at_probes(m.particle_encoder, probes, xd, 512, 16, 1), 2)
    emit(out, dict(row="end_to_end", what="estimate_mi_bounds_at_probes, notebook network, 10 000 probes, 16 x 512 sets of 50 "
                    "(409 600 particle rows encoded)", ms=round(ms_e2e, 3)))
    pm, pl = P[:20, :E].double().cpu().numpy(), P[:20, E:].double().cpu().numpy()
    dm, dl = D[:N, :E].double().cpu().numpy(), D[:N, E:].double().cpu().numpy()
    eps = rng.standard_normal((1, 20, E))
    t0 = time.perf_counter()
    PO.mi_bounds_at_probes(pm, pl, [dm], [dl], eps)
    dt = time.perf_counter() - t0
    emit(out, dict(row="cpu_baseline", what="float64 numpy oracle, 20 probes x 1 batch, extrapolated to one map",
                    nproc=os.cpu_count(), s_slice=round(dt, 3), s_per_map_extrapolated=round(dt * (M / 20) * B, 1)))


if __name__ == "__main__":
    main()
