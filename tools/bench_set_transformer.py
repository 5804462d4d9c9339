"""Time SetTransformerIBNet's training step at nb-particle cell 8's shape (12 features -> PE 5 -> [128, 128] -> E 32, sets of
50 particles, 6 blocks of 12 heads x 128, FF [128, 32], head [256] -> 1, BCE on logits) against the way the notebook's users
train it with SharedParticleEncoder: the engine encodes, a PyTorch set transformer runs forward and backward under autograd,
the engine takes d loss / d embeddings back, and two Adam updates follow (the PyTorch model exists in this tool only).

For every (precision, batch of sets) it prints one JSON line: ms per step of the library step (median of CUDA-event
intervals between consecutive graph-replayed steps), the dib_profile_* split of one eager step, the workspace bytes, and the
same median for the SharedParticleEncoder + PyTorch step ("before").  The first line names the GPU, its power limit and its
maximum SM clock.

    python tools/bench_set_transformer.py [--batches 32,256,1024] [--precisions fp32,tf32] [--steps 20] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infonce import gpu_info, profile_split  # noqa: E402

D, L, E, H, DK, BLOCKS = 12, 50, 32, 12, 128, 6


def make(precision):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(D, [128, 128], E, L, key_dim=DK, number_heads=H, number_attention_blocks=BLOCKS,
                                     precision=precision, seed=0)
    m.compile(optimizer=dib_b200.Adam(1e-4), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=["accuracy"])
    m.beta.assign(1e-3)
    return m


def data(B):
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((B, L, D)).astype(np.float32)).cuda()
    y = torch.from_numpy((rng.random((B, 1)) > 0.5).astype(np.float32)).cuda()
    return x, y


def timed(step, steps, warmup):
    for _ in range(max(warmup, 3)):                      # the library step: two eager steps, then capture and replay
        step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for i in range(steps):
        step()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]


class TorchSetTransformer(torch.nn.Module):
    """The notebook's set transformer written in PyTorch (Keras 2 MultiHeadAttention semantics, fp32)."""

    def __init__(self):
        super().__init__()
        lin = torch.nn.Linear
        self.blocks = torch.nn.ModuleList()
        for _ in range(BLOCKS):
            self.blocks.append(torch.nn.ModuleDict(dict(q=lin(E, H * DK), k=lin(E, H * DK), v=lin(E, H * DK), o=lin(H * DK, E),
                                                        ln1=torch.nn.LayerNorm(E, eps=1e-3), f1=lin(E, 128), f2=lin(128, E),
                                                        ln2=torch.nn.LayerNorm(E, eps=1e-3))))
        self.h1, self.h2 = lin(E, 256), lin(256, 1)

    def forward(self, x):
        B = x.shape[0]
        for b in self.blocks:
            sh = lambda t: t.reshape(B, L, H, DK).transpose(1, 2)
            q, k, v = sh(b["q"](x)) / math.sqrt(DK), sh(b["k"](x)), sh(b["v"](x))
            a = torch.softmax(q @ k.transpose(-1, -2), -1) @ v
            h = b["ln1"](x + b["o"](a.transpose(1, 2).reshape(B, L, H * DK)))
            x = b["ln2"](h + torch.relu(b["f2"](torch.relu(b["f1"](h)))))
        return self.h2(torch.nn.functional.leaky_relu(self.h1(x.mean(1)), 0.1))


def before_step(B, steps, warmup):
    """SharedParticleEncoder.encode -> PyTorch set transformer under autograd -> SharedParticleEncoder.gradients -> two Adams."""
    import dib_b200
    enc = dib_b200.SharedParticleEncoder(D, [128, 128], E, activation_fn='leaky_relu', leaky_alpha=0.1, seed=0)
    enc.net.optimizer.learning_rate = 1e-4
    enc.beta.assign(1e-3)
    net = TorchSetTransformer().cuda()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4, eps=1e-7)
    x, y = data(B)
    state = {"k": 0}

    def step():
        k = state["k"]
        embs, kl = enc.encode(x, step=k)
        e = embs.detach().requires_grad_(True)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(net(e), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        enc.apply_gradients(enc.gradients(x, e.grad, step=k))
        opt.step()
        state["k"] = k + 1
    return timed(step, steps, warmup)


def bench(precision, B, steps, warmup, with_before):
    m = make(precision)
    x, y = data(B)
    dts = timed(lambda: m.train_on_batch(x, y, sync=False), steps, warmup)
    res = {"precision": precision, "batch_sets": B, "particles": L, "steps": steps,
           "ms_per_step_median": round(float(np.median(dts)), 4), "ms_per_step_min": round(float(np.min(dts)), 4),
           "graph_replay": bool(m._graphs), "workspace_bytes": int(m._lib.dib_workspace_bytes(m._handle)),
           "kernel_info": m.kernel_info(B)}
    res["profile_ms"] = profile_split(m, x, y)
    del m
    torch.cuda.empty_cache()
    if with_before:
        torch.backends.cuda.matmul.allow_tf32 = precision == "tf32"
        res["before_shared_encoder_plus_torch_ms_per_step_median"] = round(float(np.median(before_step(B, steps, warmup))), 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,256,1024")
    ap.add_argument("--precisions", default="fp32,tf32")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-before", action="store_true", help="skip the SharedParticleEncoder + PyTorch comparison")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_set_transformer.py needs a CUDA device (H100)")
    lines = [json.dumps(gpu_info())]
    print(lines[-1], flush=True)
    for prec in a.precisions.split(","):
        for B in [int(b) for b in a.batches.split(",")]:
            lines.append(json.dumps(bench(prec, B, a.steps, a.warmup, not a.no_before)))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
