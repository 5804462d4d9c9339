"""Bring-up probe for the TF32 wgmma GEMM kernel: structured operands whose product reveals which element each MMA
lane actually read.  Run on the GPU box:  python tools/debug_tc_gemm.py"""
import ctypes
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from dib_b200 import _lib

lib = _lib.load()
dev = torch.device("cuda")
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
np.set_printoptions(linewidth=200, precision=1, suppress=True)


def run(mode, A, B, M, T, C, R, X=None, act=0, nsplit=1, rps=0, stride=0, simt=0, out_shape=None):
    out = torch.full(out_shape, -7.0, device=dev)
    Xp = X if X is not None else torch.zeros(4, device=dev)
    rc = lib.dib_debug_gemm_tc(mode, _lib.ptr(A), A.shape[1], _lib.ptr(B), B.shape[1], _lib.ptr(out), out.shape[-1],
                               _lib.ptr(Xp), Xp.shape[-1] if Xp.dim() > 1 else 0, M, T, C, R, act, nsplit, rps, stride, simt, st)
    if rc:
        print("ERROR:", lib.dib_last_error().decode())
    return out


def report(tag, got, want):
    got, want = got.double().cpu().numpy(), want.double().cpu().numpy()
    err = np.abs(got - want).max() / max(np.abs(want).max(), 1e-30)
    print(f"{tag}: max rel err {err:.3e}  (|want|max {np.abs(want).max():.3g}, |got|max {np.abs(got).max():.3g}, "
          f"zeros {np.mean(got == 0):.2f}, untouched {np.mean(got == -7):.2f})")
    return err


torch.manual_seed(0)
# ---------------------------------------------------------------- FWD: C = A[M,K] W[K,N] + bias(W row 0)
for (M, K, N) in [(128, 32, 128), (128, 128, 128), (96, 128, 64), (300, 512, 256)]:
    A = torch.randn(M, K, device=dev)
    W = torch.randn(K, N, device=dev)
    got = run(0, A, W, M, K, N, 0, out_shape=(M, N))
    want = A.double() @ W.double() + W[0].double()
    e = report(f"FWD  M={M} K={K} N={N}", got, want)
    ref = run(0, A, W, M, K, N, 0, simt=1, out_shape=(M, N))
    report("   simt", ref, want)
    if e > 1e-2 and K == 32:
        # structured probe: A one-hot on (r % 32), W[t][c] = 1000 t + c  -> expect (r%32)*1000 + c
        A2 = torch.zeros(M, K, device=dev)
        A2[torch.arange(M), torch.arange(M) % 32] = 1
        W2 = (torch.arange(K, device=dev)[:, None] * 1000 + torch.arange(N, device=dev)[None, :]).float()
        g2 = run(0, A2, W2, M, K, N, 0, out_shape=(M, N)) - W2[0]
        print("probe rows 0..3, cols 0..15:\n", g2[:4, :16].cpu().numpy())
        print("probe rows 30..33, cols 28..40:\n", g2[30:34, 28:40].cpu().numpy())
        print("probe row 5 all cols:\n", g2[5].cpu().numpy())

# ---------------------------------------------------------------- DGRAD: dA[M,K] = dC[M,N] W[K,N]^T
for (M, K, N) in [(128, 128, 32), (128, 128, 128), (200, 256, 64), (300, 512, 256)]:
    dC = torch.randn(M, N, device=dev)
    W = torch.randn(K, N, device=dev)
    got = run(1, dC, W, M, N, K, 0, out_shape=(M, K))
    want = dC.double() @ W.double().T
    report(f"DGRAD M={M} K={K} N={N}", got, want)

# ---------------------------------------------------------------- WGRAD: dW[K,N] = A[M,K]^T dC[M,N], db = colsum dC
for (M, K, N) in [(32, 128, 128), (256, 128, 64), (1000, 512, 256), (4096, 128, 128)]:
    A = torch.randn(M, K, device=dev)
    dC = torch.randn(M, N, device=dev)
    rps = 1024
    nsplit = (M + rps - 1) // rps
    stride = K * N + N
    out = torch.full((nsplit, stride), -7.0, device=dev)
    Xp = out.view(-1)[K * N:]                                   # db partials live right after dW inside each split
    rc = lib.dib_debug_gemm_tc(2, _lib.ptr(A), K, _lib.ptr(dC), N, _lib.ptr(out), N, _lib.ptr(Xp), 0, M, 0, N, K, 0,
                               nsplit, rps, stride, 0, st)
    if rc:
        print("ERROR:", lib.dib_last_error().decode())
    tot = out.sum(0)
    report(f"WGRAD M={M} K={K} N={N} dW", tot[:K * N].view(K, N), A.double().T @ dC.double())
    report(f"WGRAD M={M} K={K} N={N} db", tot[K * N:], dC.double().sum(0))
