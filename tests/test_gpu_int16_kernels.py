"""GPU (H100): the 16-bit integration kernels of dib_int16.cu -- the TMA + wgmma GEMM in FWD / DGRAD / WGRAD mode, the
generic and the out = 1 output head, and the fused tail -- launched through dib_debug_int16_gemm / _head / _fwd2 exactly as
the step launches them, against tests/int16_reference.py, in fp16 and bf16.

Exact cases (dyadic operands and weights, MSE with a linear output, power-of-two inv_batch, 1 / out and loss scale) must
match the float64 reference bit for bit in every output element; the reference asserts the 24-bit fit that makes that a
property of the kernels and not of luck.  The SFU activations (tanh / sigmoid / elu) and the libm losses are held to the
reference's per-element bounds; the worst measured / bound ratio is printed and collected in WORST.

Memory contracts, in every call: 16-bit NaN in every element the kernels must not read (rows >= M, pad columns, weights
past K x N, biases past N, labels and weights past n), a sentinel in every element they must not write (pad columns and
rows of the outputs, partial rows past the blocks launched, the gaps of every split slice), and the launch count.  The last
part runs the shapes no model test held to the rounding oracle through whole models."""
import ctypes

import numpy as np
import pytest
import torch

from tests import int16_reference as R
from tests.fp_exact import dyadic, from16, to16
from tests.gpu_cases import _L, _c, _grad_case, _model, _sms, _st

pytestmark = pytest.mark.gpu

FWD, DGRAD, WGRAD = 0, 1, 2
ACT = {a: i for i, a in enumerate(R.ACTS)}
LOSS = {"bce_logits": 0, "sparse_ce_logits": 1, "mse": 2, "bce_probs": 4}
FMTS = ["fp16", "bf16"]
NAN16 = {"fp16": 0x7E00, "bf16": 0x7FC0}
SENT16 = np.int16(-8531)                 # 0xDEAD: finite in both formats, never a result here
SENT32 = np.float32(-7777.25)
WORST = {}


def mat16(v, fmt, ld, extra_rows=3):
    """A [rows + extra, ld] 16-bit buffer: v in the top-left, NaN everywhere else."""
    rows, cols = v.shape
    buf = np.full((rows + extra_rows, ld), np.int16(np.uint16(NAN16[fmt]).view(np.int16)), np.int16)
    buf[:rows, :cols] = to16(v, fmt)
    return buf


def vec32(v, tail=8):
    buf = np.full(np.asarray(v).size + tail, np.nan, np.float32)
    buf[:np.asarray(v).size] = np.asarray(v, np.float32).ravel()
    return buf


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return _L().ptr(t)


class Launches:
    def __enter__(self):
        self.before = int(_L().load().dib_launch_count())
        return self

    def __exit__(self, *exc):
        self.count = int(_L().load().dib_launch_count()) - self.before


def check16(got_bits, exp, fmt, what, bound=None):
    """got_bits: a whole 16-bit output buffer; exp: the expected values of its top-left [rows, cols] block (written)."""
    rows, cols = exp.shape
    got = from16(got_bits[:rows, :cols], fmt)
    outside = np.ones(got_bits.shape, bool)
    outside[:rows, :cols] = False
    assert np.all(got_bits[outside] == SENT16), f"{what}: {int((got_bits[outside] != SENT16).sum())} elements written outside"
    _compare(got, got_bits[:rows, :cols], exp, bound, what, lambda v: to16(v, fmt))


def check32(got, exp, what, bound=None):
    """got: a whole fp32 buffer; exp: its expected leading values; the rest must hold the sentinel."""
    exp = np.asarray(exp, np.float64).ravel()
    assert np.all(got[exp.size:] == SENT32), f"{what}: {int((got[exp.size:] != SENT32).sum())} floats written outside"
    _compare(got[:exp.size].astype(np.float64), got[:exp.size].view(np.uint32), exp,
             None if bound is None else np.asarray(bound).ravel(), what, lambda v: np.asarray(v, np.float32).view(np.uint32))


def _compare(got, got_bits, exp, bound, what, to_bits):
    """An exact output (no bound) must carry the expected bit pattern in every element, so a zero of the wrong sign fails
    too; a bounded output must lie within its bound, and its elements with a zero bound must equal the reference."""
    assert np.isfinite(got).all() or np.array_equal(np.isnan(got), np.isnan(exp)), f"{what}: a NaN operand was read"
    if bound is None or not np.any(bound):
        live = ~(np.isnan(got) & np.isnan(exp))
        want = to_bits(np.where(live, exp, 0.0))
        if not np.array_equal(got_bits[live], want[live]):
            bad = np.argwhere(live & (got_bits != want))
            i = tuple(bad[0])
            raise AssertionError(f"{what}: {len(bad)} elements differ, first at {i}: got {got[i]!r} (bits {got_bits[i]:#x}), "
                                 f"want {exp[i]!r} (bits {want[i]:#x})")
        return
    err = np.abs(got - exp)
    ok = (err <= bound) | (np.isnan(got) & np.isnan(exp))
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements outside the bound, first at {i}: got {got[i]!r}, want "
                             f"{exp[i]!r} +- {bound[i]!r}")
    # the exact elements of a bounded output (a zero act') are compared by value: the sign of such a zero follows the sign
    # of an inexact sum
    exact = (bound == 0) & np.isfinite(exp)
    if exact.any():
        assert np.array_equal(got[exact], exp[exact]), f"{what}: an exact element differs"
    inexact = ~exact & np.isfinite(err)
    if inexact.any():
        r = float((err[inexact] / bound[inexact]).max())
        WORST[what.split(" ")[0]] = max(WORST.get(what.split(" ")[0], 0.0), r)


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
def run_fwd(fmt, M, K, N, act="relu", alpha=0.25, seed=0, scale=1.0, bias_scale=None):
    rng = np.random.default_rng(seed)
    a, w = dyadic(rng, (M, K)) * scale, dyadic(rng, (K, N)) * scale
    b = dyadic(rng, (N,)) * (scale * scale if bias_scale is None else bias_scale)
    lda, ldc = K + 8, N + 8
    nan = np.int16(np.uint16(NAN16[fmt]).view(np.int16))
    A, W = dev(mat16(a, fmt, lda)), dev(np.concatenate([mat16(w, fmt, N, 0).ravel(), np.full(64, nan, np.int16)]))
    B = dev(vec32(b))
    out = dev(np.full((M + 3, ldc), SENT16, np.int16))
    with Launches() as n:
        _L().check(_L().load().dib_debug_int16_gemm(FWD, fmt == "bf16", M, K, N, ptr(A), lda, ptr(W), ptr(B), None, 0, ptr(out),
                                                    ldc, ACT[act], alpha, None, None, 0, 0, 1.0, _st()))
    assert n.count == 1
    exp, bound = R.gemm_fwd(a, w, b, act, alpha, fmt)
    check16(out.cpu().numpy(), exp, fmt, f"fwd {fmt} {act} M={M} K={K} N={N}", bound)
    return exp


def run_dgrad(fmt, M, K, N, act="relu", alpha=0.25, seed=0, with_x=True, with_colsum=True):
    rng = np.random.default_rng(seed)
    dz, w = dyadic(rng, (M, N)), dyadic(rng, (K, N))
    x = (rng.integers(-15, 16, size=(M, K)) / 16).astype(np.float64)
    if act == "relu":
        x = np.maximum(x, 0.0)                               # relu outputs are >= 0
    lda, ldc, ldx = N + 8, K + 16, K + 8
    nan = np.int16(np.uint16(NAN16[fmt]).view(np.int16))
    A = dev(mat16(dz, fmt, lda))
    W = dev(np.concatenate([mat16(w, fmt, N, 0).ravel(), np.full(64, nan, np.int16)]))
    X = dev(mat16(x, fmt, ldx)) if with_x else None
    out = dev(np.full((M + 3, ldc), SENT16, np.int16))
    tiles = -(-M // 128)
    cs = dev(np.full((tiles + 1) * K, SENT32, np.float32)) if with_colsum else None
    with Launches() as n:
        _L().check(_L().load().dib_debug_int16_gemm(DGRAD, fmt == "bf16", M, K, N, ptr(A), lda, ptr(W), None, ptr(X),
                                                    ldx, ptr(out), ldc, ACT[act], alpha, ptr(cs), None, 0, 0, 1.0, _st()))
    assert n.count == 1
    exp, colsum = R.gemm_dgrad(dz, w, x if with_x else None, act, alpha, fmt)
    check16(out.cpu().numpy(), exp, fmt, f"dgrad {fmt} {act} M={M} K={K} N={N}")
    if with_colsum:
        check32(cs.cpu().numpy(), colsum, f"dgrad-colsum {fmt} M={M} K={K}")


def run_wgrad(fmt, M, layers, out_scale=0.25, seed=0):
    """layers: [(K, N, nsplit, rps)], one or two; both layers' partials in one buffer at the step's layout (one split row
    of split_stride floats holds every layer's [K x N] block, sentinel gaps between them)."""
    rng = np.random.default_rng(seed)
    offs, o = [], 0
    for K, N, _, _ in layers:
        offs.append(o)
        o += K * N + 64
    ss = o + 32
    nsplit_max = max(l[2] for l in layers)
    part = dev(np.full(ss * nsplit_max + 64, SENT32, np.float32))
    descs = (_L().DibInt16WgradLayer * len(layers))()
    keep, exp = [], np.full(ss * nsplit_max + 64, SENT32, np.float64)
    for q, (K, N, nsplit, rps) in enumerate(layers):
        g, dz = dyadic(rng, (M, K)), dyadic(rng, (M, N))
        G, D = dev(mat16(g, fmt, K)), dev(mat16(dz, fmt, N))
        keep += [G, D]
        d = descs[q]
        d.g_in, d.K, d.dz, d.N = G.data_ptr(), K, D.data_ptr(), N
        d.dW_part, d.nsplit, d.rows_per_split = part.data_ptr() + 4 * offs[q], nsplit, rps
        ref = R.gemm_wgrad(g, dz, M, nsplit, rps, out_scale)
        for s in range(nsplit):
            exp[s * ss + offs[q]:s * ss + offs[q] + K * N] = ref[s].ravel()
    with Launches() as n:
        _L().check(_L().load().dib_debug_int16_gemm(WGRAD, fmt == "bf16", M, 0, 0, None, 0, None, None, None, 0, None, 0, 0, 0.0,
                                                    None, descs, len(layers), ss, out_scale, _st()))
    assert n.count == 1
    got = part.cpu().numpy().astype(np.float64)
    if not np.array_equal(got, exp):
        i = int(np.flatnonzero(got != exp)[0])
        raise AssertionError(f"wgrad {fmt} M={M} {layers}: {int((got != exp).sum())} floats differ, first at {i} (split "
                             f"{i // ss}, offset {i % ss}): got {got[i]}, want {exp[i]}")


GEMM_M = [1, 63, 64, 65, 127, 128, 129, 4097]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M", GEMM_M)
def test_fwd_rows(fmt, M):
    for K, N in ((64, 128), (192, 256), (320, 384), (512, 512)):
        run_fwd(fmt, M, K, N, "leaky_relu", 0.25, seed=M + K)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("K", [64, 128, 192, 256, 320, 512, 1024])
@pytest.mark.parametrize("N", [128, 256, 384, 512])
def test_fwd_widths(fmt, K, N):
    run_fwd(fmt, 129, K, N, "relu", seed=K + N)


@pytest.mark.parametrize("fmt", FMTS)
def test_fwd_many_tiles(fmt):
    """More tiles than 2 x SMs: every CTA walks several tiles and carries the ring's phase across them."""
    M = 128 * (2 * _sms() + 5) + 17
    run_fwd(fmt, M, 320, 384, "linear", seed=3)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act,alpha", [(a, al) for a in R.ACTS for al in ((0.25, 0.2) if a == "leaky_relu" else (0.2,))])
def test_fwd_activations(fmt, act, alpha):
    run_fwd(fmt, 257, 192, 256, act, alpha, seed=ACT[act])


@pytest.mark.parametrize("fmt", FMTS)
def test_fwd_saturation_and_subnormals(fmt):
    """Pre-activations beyond 65 504 (cvt.rn.satfinite gives +-65 504 in fp16) and results in fp16's subnormal range."""
    big = run_fwd(fmt, 129, 1024, 128, "linear", scale=64.0, seed=11)
    if fmt == "fp16":
        assert np.abs(big).max() == 65504.0
    tiny = run_fwd(fmt, 129, 256, 128, "leaky_relu", 0.25, scale=2.0 ** -12, seed=12)
    if fmt == "fp16":
        assert np.any((tiny != 0) & (np.abs(tiny) < 2.0 ** -14))


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M", GEMM_M)
def test_dgrad_rows(fmt, M):
    for K, N in ((64, 128), (192, 256), (320, 384), (512, 256)):
        run_dgrad(fmt, M, K, N, "leaky_relu", 0.2, seed=M + K)
        run_dgrad(fmt, M, K, N, "linear", seed=M + K + 1, with_x=False)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act", R.ACTS)
def test_dgrad_activations(fmt, act):
    run_dgrad(fmt, 300, 192, 256, act, 0.25, seed=20 + ACT[act])
    run_dgrad(fmt, 129, 320, 128, act, 0.2, seed=30 + ACT[act], with_colsum=False)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,rps,extra", [(1, 64, 0), (129, 64, 0), (1000, 256, 0), (1000, 320, 2), (4097, 256, 1),
                                         (4097, 1024, 0)])
def test_wgrad_one_layer(fmt, M, rps, extra):
    """rows_per_split 64 / 256 / 320, a short last split and splits past the batch (zero partials); R = K = 192 / 320."""
    for K, N in ((192, 256), (320, 128)):
        run_wgrad(fmt, M, [(K, N, -(-M // rps) + extra, rps)], seed=M + K)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M", [129, 1000, 4097])
def test_wgrad_two_layers(fmt, M):
    """Two layers of different shapes and split counts in one launch."""
    run_wgrad(fmt, M, [(192, 256, -(-M // 64), 64), (256, 384, -(-M // 320) + 1, 320)], seed=M)
    run_wgrad(fmt, M, [(512, 128, -(-M // 256), 256), (64, 256, 2 * -(-M // 1024), 1024)], out_scale=2.0 ** -10, seed=M + 1)


# ---------------------------------------------------------------------------------------------------------------------
# output heads
# ---------------------------------------------------------------------------------------------------------------------
def run_head(fmt, n, out, nblocks, loss="mse", out_act="linear", hid_act="relu", head1=False, weighted=False, train=True,
             with_y=True, seed=0, alpha=0.25):
    rng = np.random.default_rng(seed)
    K = 256
    g = dyadic(rng, (n, K), k=2, den=2)
    if hid_act == "relu":
        g = np.maximum(g, 0)
    elif hid_act in ("tanh", "sigmoid", "elu"):
        g = (rng.integers(-7, 8, size=(n, K)) / 8).astype(np.float64) * (0.5 if hid_act == "sigmoid" else 1)
        if hid_act == "sigmoid":
            g = np.abs(g)
    Wc, bc = dyadic(rng, (K, out), k=1, den=8), dyadic(rng, (out,), k=4, den=16)
    exact = loss == "mse" and out_act == "linear" and (out & (out - 1)) == 0
    if loss == "sparse_ce_logits":
        y = rng.integers(0, out, size=n).astype(np.float64)
        edge = [0.0, out - 1.0, -0.5, min(out - 1, 2) + 0.5]      # 0, C - 1, -0.5 (class 0), 2.5 (class 2, never a hit)
        y[:min(n, 4)] = edge[:min(n, 4)]
    elif loss == "mse":
        y = g @ Wc + bc + dyadic(rng, (n, out), k=2, den=16)        # small residuals: every loss sum fits 24 bits
    else:
        y = rng.integers(0, 2, size=(n, out)).astype(np.float64)
    w = dyadic(rng, (n,), k=4, den=2) + 2.5 if weighted else None        # in [0.5, 4.5], dyadic
    ib = 2.0 ** -int(np.ceil(np.log2(n)))
    S = 2.0 ** 7
    ldg = K + 8
    G = dev(mat16(g, fmt, ldg))
    Wd, Bd = dev(vec32(Wc)), dev(vec32(bc))
    Y = dev(vec32(y)) if with_y else None
    Wt = dev(vec32(w)) if weighted else None
    stride = K * out + out + K + 5
    dg = dev(np.full((n + 3, ldg), SENT16, np.int16)) if train else None
    up = dev(np.full(n * out + 8, SENT32, np.float32))
    wp = dev(np.full(nblocks * stride + 8, SENT32, np.float32)) if train else None
    lp, ap = (dev(np.full(nblocks + 4, SENT32, np.float32)) for _ in range(2))
    with Launches() as c:
        _L().check(_L().load().dib_debug_int16_head(int(head1), fmt == "bf16", ptr(G), ldg, K, ptr(Wd), ptr(Bd), out, ACT[out_act],
                                                    ACT[hid_act], alpha, LOSS[loss], ptr(Y), n, ib, S, ptr(dg), ldg, ptr(up),
                                                    ptr(wp), stride, ptr(lp), ptr(ap), nblocks, ptr(Wt), _st()))
    assert c.count == 1
    zk = up.cpu().numpy()
    ref = R.head(g, Wc, bc, out_act, hid_act, alpha, loss, y if with_y else None, ib, S, w, nblocks, head1, fmt,
                 z_kernel=zk[:n * out].astype(np.float64), train=train, exact=exact)
    tag = f"{fmt} {'head1' if head1 else 'head'} n={n} out={out} nb={nblocks} {loss} {hid_act}"
    check32(zk, ref["z"], "head-z " + tag, ref["z_bound"])
    check32(lp.cpu().numpy(), ref["loss_part"], "head-loss " + tag, ref["loss_part_bound"])
    check32(ap.cpu().numpy(), ref["acc_part"], "head-acc " + tag, ref["acc_part_bound"])
    if train:
        check16(dg.cpu().numpy(), ref["dg"], fmt, "head-dg " + tag, ref["dg_bound"])
        full = np.full((nblocks, stride), SENT32, np.float64)
        full[:, :ref["wpart"].shape[1]] = ref["wpart"]
        fb = np.zeros_like(full)
        fb[:, :ref["wpart"].shape[1]] = ref["wpart_bound"]
        check32(wp.cpu().numpy(), full, "head-wpart " + tag, fb)
    return ref


HEAD_N = [1, 3, 4, 5, 255, 256, 257, 20001]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("out", [1, 2, 3, 4, 5, 8, 9, 16])
@pytest.mark.parametrize("n", HEAD_N)
def test_head_exact(fmt, out, n):
    """MSE with a linear output: bit for bit for out a power of two; out 3, 5, 9 round 1 / out and carry bounds."""
    for nb in (1, 3, 2 * _sms()):
        run_head(fmt, n, out, nb, seed=n + out + nb, weighted=nb == 3)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("n", HEAD_N)
def test_head1_exact(fmt, n):
    for nb in (1, 3, 2 * _sms()):
        run_head(fmt, n, 1, nb, head1=True, seed=n + nb, weighted=nb == 3)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("head1", [False, True])
@pytest.mark.parametrize("hid_act", R.ACTS)
def test_head_hidden_activations(fmt, head1, hid_act):
    """act'(h) from the 16-bit h is exact on the 1/8 grid for every activation: bit for bit."""
    for out in ((1,) if head1 else (2, 16)):
        for weighted in (False, True):
            run_head(fmt, 257, out, 3, hid_act=hid_act, head1=head1, weighted=weighted, seed=ACT[hid_act] + out)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("head1", [False, True])
@pytest.mark.parametrize("loss,out_act", [("bce_logits", "linear"), ("sparse_ce_logits", "linear"), ("bce_probs", "sigmoid")])
def test_head_losses(fmt, head1, loss, out_act):
    """The libm losses, held to the per-element bounds of tests/elementwise_reference.loss on the kernel's z."""
    for out in ((1,) if head1 else (1, 3, 9, 16)):
        for n in (5, 257, 4097):
            run_head(fmt, n, out, 3, loss=loss, out_act=out_act, head1=head1, weighted=n == 257, seed=n + out)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("head1", [False, True])
def test_head_inference_and_no_labels(fmt, head1):
    out = 1 if head1 else 5
    run_head(fmt, 257, out, 3, head1=head1, train=False)                   # inference: no dg, no partials
    run_head(fmt, 257, out, 3, head1=head1, with_y=False)                  # y = null: zero gradients
    run_head(fmt, 257, out, 3, head1=head1, with_y=False, train=False)


# ---------------------------------------------------------------------------------------------------------------------
# the fused tail
# ---------------------------------------------------------------------------------------------------------------------
def run_fwd2(fmt, M, K0, act="relu", stages=3, demb=False, weighted=False, seed=0, alpha=0.25, with_y=True):
    rng = np.random.default_rng(seed)
    a = dyadic(rng, (M, K0), k=2, den=2)
    W0, W1 = dyadic(rng, (K0, 256), k=1, den=8), dyadic(rng, (256, 256), k=1, den=8)
    b0, b1 = dyadic(rng, (256,), k=2, den=8), dyadic(rng, (256,), k=2, den=8)
    wout, bout = dyadic(rng, (256,), k=2, den=8), np.array([0.125])
    sfu = act in ("tanh", "sigmoid", "elu")
    if sfu:
        y = dyadic(rng, (M, 1), k=4, den=4)
    else:
        z = R.fwd2(a, W0, b0, W1, b1, wout, bout, act, alpha, None, 1.0, 1.0, 1, fmt, stages=1)["z"]
        y = z[:, None] + dyadic(rng, (M, 1), k=2, den=16)             # small residuals: every loss sum fits 24 bits
    w = dyadic(rng, (M,), k=4, den=2) + 2.5 if weighted else None
    ib, S = 2.0 ** -int(np.ceil(np.log2(M))), 2.0 ** 7
    nan = np.int16(np.uint16(NAN16[fmt]).view(np.int16))
    A = dev(mat16(a, fmt, K0 + 8))
    W0d = dev(np.concatenate([mat16(W0, fmt, 256, 0).ravel(), np.full(64, nan, np.int16)]))
    W1d = dev(np.concatenate([mat16(W1, fmt, 256, 0).ravel(), np.full(64, nan, np.int16)]))
    b0d, b1d, wod, bod = (dev(vec32(v)) for v in (b0, b1, wout, bout))
    Y = dev(vec32(y)) if with_y else None
    Wt = dev(vec32(w)) if weighted else None
    sent = lambda rows, cols: dev(np.full((rows, cols), SENT16, np.int16))
    g1 = sent(M + 3, 256)
    dg2 = sent(M + 3, 256) if stages >= 2 else None
    dg1 = sent(M + 3, 256) if stages >= 3 else None
    de = sent(M + 3, K0) if demb else None
    tiles = -(-M // 128)
    dbp = dev(np.full((tiles + 1) * 256, SENT32, np.float32)) if stages >= 3 else None
    grid_max = _sms()
    up = dev(np.full(M + 8, SENT32, np.float32))
    stride = 2 * 256 + 1 + 3
    wp = dev(np.full(grid_max * stride + 8, SENT32, np.float32)) if stages >= 2 else None
    lp, ap = (dev(np.full(grid_max + 4, SENT32, np.float32)) for _ in range(2))
    nb = ctypes.c_int32(-1)
    with Launches() as c:
        _L().check(_L().load().dib_debug_int16_fwd2(fmt == "bf16", ptr(A), K0 + 8, K0, ptr(W0d), ptr(b0d), ptr(W1d), ptr(b1d), ptr(g1),
                                                    ptr(wod), ptr(bod), ACT[act], ACT["linear"], alpha, LOSS["mse"], ptr(Y), M,
                                                    ib, S, ptr(dg2), ptr(dg1), ptr(dbp), ptr(de), ptr(up), ptr(wp), stride,
                                                    ptr(lp), ptr(ap), ptr(Wt), ctypes.byref(nb), _st()))
    assert c.count == 1
    out = dict(g1=g1.cpu().numpy(), z=up.cpu().numpy(), loss=lp.cpu().numpy(), acc=ap.cpu().numpy())
    out.update(dg2=dg2.cpu().numpy() if dg2 is not None else None, dg1=dg1.cpu().numpy() if dg1 is not None else None,
               wpart=wp.cpu().numpy() if wp is not None else None, dbpart=dbp.cpu().numpy() if dbp is not None else None,
               demb=de.cpu().numpy() if de is not None else None)
    yy = y if with_y else None
    if sfu:
        # every stage after g1 continues from the kernel's own stored intermediates
        kern = dict(g1=from16(out["g1"][:M], fmt), z=out["z"][:M].astype(np.float64))
        if stages >= 2:
            kern["dg2"] = from16(out["dg2"][:M], fmt)
        if stages >= 3:
            kern["dg1"] = from16(out["dg1"][:M], fmt)
        ref = R.fwd2_sfu(a, W0, b0, W1, b1, wout, bout, act, alpha, yy, ib, S, grid_max, fmt, kern, w, stages, demb)
    else:
        ref = R.fwd2(a, W0, b0, W1, b1, wout, bout, act, alpha, yy, ib, S, grid_max, fmt, w, stages, demb)
    bnd = lambda k: ref.get(k + "_bound")
    grid = ref["grid"]
    assert nb.value == grid
    tag = f"{fmt} M={M} K0={K0} {act} stages={stages} demb={demb} w={weighted}"
    check16(out["g1"], ref["g1"], fmt, "tail-g1 " + tag, bnd("g1"))
    check32(out["z"], ref["z"], "tail-z " + tag, bnd("z"))
    check32(out["loss"], ref["loss_part"], "tail-loss " + tag, bnd("loss_part"))
    check32(out["acc"], ref["acc_part"], "tail-acc " + tag, bnd("acc_part"))
    if stages >= 2:
        check16(out["dg2"], ref["dg2"], fmt, "tail-dg2 " + tag, bnd("dg2"))
        full = np.full((grid, stride), SENT32, np.float64)
        full[:, :513] = ref["wpart"]
        fb = None
        if bnd("wpart") is not None:
            fb = np.zeros_like(full)
            fb[:, :513] = bnd("wpart")
        check32(out["wpart"], full, "tail-wpart " + tag, fb)
    if stages >= 3:
        check16(out["dg1"], ref["dg1"], fmt, "tail-dg1 " + tag, bnd("dg1"))
        check32(out["dbpart"], ref["dbpart"], "tail-dbpart " + tag, bnd("dbpart"))
    if demb:
        check16(out["demb"], ref["demb"], fmt, "tail-demb " + tag, bnd("demb"))


TAIL_STAGES = [(1, False), (2, False), (3, False), (3, True)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("K0", [64, 128, 192, 256, 320, 512])
@pytest.mark.parametrize("stages,demb", TAIL_STAGES)
def test_fwd2_widths(fmt, K0, stages, demb):
    for M in (1, 129):
        run_fwd2(fmt, M, K0, "leaky_relu", stages, demb, seed=K0 + M)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("Mk", ["1", "127", "128", "129", "sms+1", "2sms+77"])
def test_fwd2_rows(fmt, Mk):
    """Up to 256 SMs + 77 rows: every CTA runs two or three tiles and carries the ring's phase."""
    M = {"sms+1": 128 * _sms() + 1, "2sms+77": 256 * _sms() + 77}.get(Mk) or int(Mk)
    for weighted in (False, True):
        run_fwd2(fmt, M, 320, "relu", 3, True, weighted=weighted, seed=M)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act", R.ACTS)
@pytest.mark.parametrize("stages,demb", TAIL_STAGES)
def test_fwd2_activations(fmt, act, stages, demb):
    """linear / relu / leaky ReLU bit for bit; tanh / sigmoid / elu (the SFU instantiations) within the reference's bounds,
    each stage judged on the kernel's own stored inputs."""
    for weighted in (False, True):
        run_fwd2(fmt, 257, 192, act, stages, demb, weighted=weighted, seed=ACT[act])


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act", ["tanh", "sigmoid", "elu"])
def test_fwd2_sfu_shapes(fmt, act):
    """The SFU instantiations at K0 = 320 (three d emb chunks, the last half full) and at several CTAs' worth of tiles."""
    run_fwd2(fmt, 129, 320, act, 3, True, seed=40 + ACT[act])
    run_fwd2(fmt, 128 * _sms() + 1, 320, act, 3, True, weighted=True, seed=50 + ACT[act])


@pytest.mark.parametrize("fmt", FMTS)
def test_fwd2_no_labels(fmt):
    run_fwd2(fmt, 257, 192, "relu", 3, True, with_y=False)


# ---------------------------------------------------------------------------------------------------------------------
# the hooks refuse bad arguments on the host (nothing is launched)
# ---------------------------------------------------------------------------------------------------------------------
def _refused(fn, match, **kw):
    with Launches() as c:
        with pytest.raises(_L().DibError, match=match):
            _L().check(fn(**kw))
    assert c.count == 0


def test_hooks_refuse_bad_arguments():
    lib = _L().load()
    buf = torch.zeros(1 << 20, dtype=torch.int16, device="cuda")
    f32b = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    p, q = ptr(buf), ptr(f32b)
    odd = ctypes.c_void_p(buf.data_ptr() + 2)
    st = _st()
    gemm = lambda mode=FWD, M=128, K=64, N=128, a=p, lda=64, bias=q, ldc=128, **kw: lib.dib_debug_int16_gemm(
        mode, 0, M, K, N, a, lda, p, bias, kw.get("x"), kw.get("ldx", 0), p, ldc, 1, 0.2, None, kw.get("layers"),
        kw.get("count", 0), kw.get("ss", 0), 1.0, st)
    _refused(gemm, K=96, match="K a positive multiple of 64")
    _refused(gemm, N=192, match="N a positive multiple of 128")
    _refused(gemm, M=0, match="M >= 1")
    _refused(gemm, lda=60, match="lda must be a multiple of 8")
    _refused(gemm, lda=72 - 4, match="lda")
    _refused(gemm, ldc=120, match="ldc")
    _refused(gemm, a=odd, match="a must be 16-byte aligned")
    _refused(gemm, bias=ctypes.c_void_p(f32b.data_ptr() + 4), match="bias must be 8-byte aligned")
    _refused(gemm, bias=None, match="FWD needs bias")
    _refused(gemm, mode=DGRAD, lda=128, ldc=64, x=p, ldx=32, match="ldx")

    def wg(K=192, N=256, nsplit=2, rps=64, M=128, ss=192 * 256, count=1):
        L = (_L().DibInt16WgradLayer * 2)()
        for l in L:
            l.g_in, l.K, l.dz, l.N, l.dW_part, l.nsplit, l.rows_per_split = buf.data_ptr(), K, buf.data_ptr(), N, f32b.data_ptr(), nsplit, rps
        return gemm(mode=WGRAD, M=M, layers=L, count=count, ss=ss)
    _refused(wg, rps=32, match="rows_per_split a positive multiple of 64")
    _refused(wg, rps=96, match="rows_per_split a positive multiple of 64")
    _refused(wg, nsplit=1, M=65, match=r"nsplit \* rows_per_split >= M")
    _refused(wg, ss=192 * 256 - 2, match="inside split_stride")
    _refused(wg, count=3, match="1 or 2 layers")
    _refused(wg, K=100, match="K a positive multiple of 64")

    def hd(head1=0, K=256, out=1, ldg=256, stride=513, n=10, nblocks=1, g=p, dg=p, loss=2):
        return lib.dib_debug_int16_head(head1, 0, g, ldg, K, q, q, out, 0, 1, 0.2, loss, q, n, 1.0, 1.0, dg, ldg, None, q,
                                        stride, q, q, nblocks, None, st)
    _refused(hd, K=128, match="K == 256")
    _refused(hd, out=17, match="1 <= out_dim <= 16")
    _refused(hd, out=0, match="1 <= out_dim <= 16")
    _refused(hd, head1=1, out=2, stride=2 * 256 + 2 + 256, match="head1 needs out_dim == 1")
    _refused(hd, stride=512, match="wpart_stride >= K \\* out_dim \\+ out_dim \\+ K")
    _refused(hd, ldg=260, match="ldg")
    _refused(hd, g=odd, match="g must be 16-byte aligned")
    _refused(hd, nblocks=0, match="nblocks")
    _refused(hd, loss=3, match="unknown loss")

    def tl(K0=192, dg2=p, dg1=p, dbpart=q, demb=p, stride=513, ld_in=192, M=10):
        nb = ctypes.c_int32(0)
        return lib.dib_debug_int16_fwd2(0, p, ld_in, K0, p, q, p, q, p, q, q, 1, 0, 0.2, 2, q, M, 1.0, 1.0, dg2, dg1, dbpart,
                                        demb, None, q, stride, q, q, None, ctypes.byref(nb), st)
    _refused(tl, K0=96, match="K0 a positive multiple of 64")
    _refused(tl, K0=0, ld_in=8, match="K0 a positive multiple of 64")
    _refused(tl, dg2=None, match="dg1 needs dg2 and dbpart")
    _refused(tl, dbpart=None, match="dg1 needs dg2 and dbpart")
    _refused(tl, dg1=None, match="demb needs dg1")
    _refused(tl, stride=512, match="wpart_stride >= 513")
    _refused(tl, ld_in=188, match="ld_in")


# ---------------------------------------------------------------------------------------------------------------------
# whole models: the shapes no model test held to the rounding oracle (the harness and bounds of
# test_gpu_fused16_vs_rounding_oracle.py)
# ---------------------------------------------------------------------------------------------------------------------
MODEL_SHAPES = {
    "F6_tail": (dict(F=6), "relu", 0, "dgrad"),                  # K0 = 192: a half-full last d emb chunk at c0 = 128
    "F10_tail": (dict(F=10), "relu", 0, "dgrad"),                # K0 = 320: three d emb chunks, the last half full
    # one hidden layer and no fused tail: the head1 kernel, and the backward's DGRAD to the embedding and lone layer-0 WGRAD
    # (R = 192) that a one-layer integration network without a tail runs
    "F6_head1": (dict(F=6, integ=(256,)), "relu", 0, None),
    "F10_384": (dict(F=10, integ=(384, 256)), "relu", 0, None),  # a 384-wide layer: three column tiles, head1
    "sigmoid_tail": (dict(F=6), "sigmoid", 0, "dgrad"),
    "elu_tail": (dict(F=10), "elu", 0, "dgrad"),
}


@pytest.mark.parametrize("prec", FMTS)
@pytest.mark.parametrize("shape", list(MODEL_SHAPES))
def test_model_shapes_against_rounding_oracle(shape, prec):
    kw, act, mask, tail = MODEL_SHAPES[shape]
    cfg = _c(act=act, **kw)
    n = 128 * 20 + 77
    if tail is None:                                 # no fused tail: the out = 1 head kernel
        info = _model(cfg, prec, "bce_logits", mask).kernel_info(n)
        assert "integration_head=head1" in info, info
    _grad_case(cfg, prec, "bce_logits", n, 1e-3, seed=7, mask=mask, tail=tail, label=shape)


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratios():
    """A report, not a check (_compare checks every element): after the module, the worst measured / bound ratio of every
    bounded output kind compared in this process."""
    yield
    for k, v in sorted(WORST.items()):
        print(f"\n[int16-kernels] worst measured / bound {k}: {v:.3f}")
