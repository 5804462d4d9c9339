"""CPU: tests/int16_reference.py, the float64 reference of the 16-bit integration kernels -- without rounding it is the model
oracle's arithmetic, its generators and exactness claims hold, and every seeded kernel fault breaks the exact comparison."""
import numpy as np
import pytest

from oracle import dib_oracle as O
from tests import fused16_oracle as Q
from tests import int16_reference as R
from tests.fp_exact import FORMATS, dyadic, exact_matmul, quantum, ulp16

FMTS = ["fp16", "bf16"]


def _layers(seed, M=300, K0=192):
    rng = np.random.default_rng(seed)
    a = dyadic(rng, (M, K0), k=2, den=2)
    W0, W1 = dyadic(rng, (K0, 256), k=1, den=8), dyadic(rng, (256, 256), k=1, den=8)
    b0, b1 = dyadic(rng, (256,), k=2, den=8), dyadic(rng, (256,), k=2, den=8)
    wout, bout = dyadic(rng, (256,), k=2, den=8), np.array([0.125])
    return a, W0, b0, W1, b1, wout, bout


def _same(x, y):
    return np.array_equal(np.asarray(x, np.float64), np.asarray(y, np.float64))


# ---- without rounding the reference is the oracle's arithmetic ----------------------------------------------------------
@pytest.mark.parametrize("act", ["linear", "relu", "leaky_relu"])
def test_unrounded_tail_is_the_oracle(act):
    """fmt None: the fused tail's g1, logit, dg2, dg1 and d emb are the float64 layer formulas of dib_oracle /
    fused16_oracle (forward: g = act(g W + b); backward: d = (S dz) w act'(g), then d W^T act'(g))."""
    a, W0, b0, W1, b1, wout, bout = _layers(1)
    alpha, M = 0.25, a.shape[0]
    z0 = R.fwd2(a, W0, b0, W1, b1, wout, bout, act, alpha, None, 1.0, 1.0, 4, None, stages=1)["z"]
    y = z0[:, None] + 0.125
    ib, S = 2.0 ** -9, 2.0 ** 9
    ref = R.fwd2(a, W0, b0, W1, b1, wout, bout, act, alpha, y, ib, S, 4, None, stages=3, demb=True)
    g1 = O.act_fwd(act, a @ W0 + b0, alpha)
    g2 = O.act_fwd(act, g1 @ W1 + b1, alpha)
    z = g2 @ wout + bout[0]
    assert _same(ref["g1"], g1) and _same(ref["z"], z)
    dzs = O.task_loss_grad(O.LOSS_MSE, z[:, None], y)[:, 0] * ib
    assert np.allclose(dzs, 2 * (z - y[:, 0]) * ib)
    d2 = (S * dzs)[:, None] * wout[None, :] * O.act_grad_from_output(act, g2, alpha)
    assert _same(ref["dg2"], d2)
    d1 = (d2 @ W1.T) * O.act_grad_from_output(act, g1, alpha)
    assert _same(ref["dg1"], d1) and _same(ref["demb"], d1 @ W0.T)
    tiles = -(-M // 128)
    assert np.allclose(ref["dbpart"].sum(0), d1.sum(0), rtol=0, atol=1e-9) and ref["dbpart"].shape == (tiles, 256)
    assert np.isclose(ref["loss_part"].sum(), ((z - y[:, 0]) ** 2).sum())
    assert np.allclose(ref["wpart"].sum(0)[:256], g2.T @ dzs) and np.isclose(ref["wpart"][:, 256].sum(), dzs.sum())


def test_unrounded_gemms_and_head_are_the_oracle():
    rng = np.random.default_rng(2)
    a, w, b = dyadic(rng, (200, 192)), dyadic(rng, (192, 256)), dyadic(rng, (256,))
    for act in ("linear", "relu", "leaky_relu"):
        assert _same(R.gemm_fwd(a, w, b, act, 0.25, None)[0], O.act_fwd(act, a @ w + b, 0.25))
    x = (rng.integers(-15, 16, size=(200, 192)) / 16)
    dz = dyadic(rng, (200, 256))
    for act in R.ACTS:
        out, cs = R.gemm_dgrad(dz, w, x, act, 0.25, None)
        assert _same(out, (dz @ w.T) * O.act_grad_from_output(act, x, 0.25))
        assert np.allclose(cs.sum(0), out.sum(0), rtol=0, atol=1e-9)
    parts = R.gemm_wgrad(a, dz, 200, 5, 64, 0.5)                     # split 4 lies past the batch: zeros
    assert _same(parts.sum(0), 0.5 * a.T @ dz) and not parts[4].any()
    g = np.maximum(dyadic(rng, (300, 256), k=2, den=2), 0)
    Wc, bc = dyadic(rng, (256, 4), k=1, den=8), dyadic(rng, (4,), k=4, den=16)
    y = g @ Wc + bc + 0.0625
    h = R.head(g, Wc, bc, "linear", "relu", 0.2, "mse", y, 2.0 ** -9, 2.0 ** 9, nblocks=3, fmt=None, exact=True)
    dz = O.task_loss_grad(O.LOSS_MSE, g @ Wc + bc, y) * 2.0 ** -9
    assert _same(h["dg"], 2.0 ** 9 * (dz @ Wc.T) * (g > 0))
    assert np.allclose(h["wpart"].sum(0)[:1024], (g.T @ dz).ravel(), rtol=0, atol=1e-12)


# ---- the generators are exact -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_generators_are_exact(fmt):
    rng = np.random.default_rng(3)
    for k, den in ((4, 4), (2, 2), (1, 8), (2, 16)):
        v = dyadic(rng, (1000,), k, den)
        assert _same(Q.round_to(v, fmt), v) and quantum(v) >= 1.0 / den
    assert quantum([0.75, 3.0, 3 * 2.0 ** -20]) == 2.0 ** -20 and quantum([0.0]) == 1.0
    with pytest.raises(AssertionError, match="24 bits"):
        exact_matmul(np.full((1, 2 ** 13), 0.25), np.full((2 ** 13, 1), 2.0 ** 10 + 0.25), "sum")
    exact_matmul(np.full((1, 256), 0.25), np.full((256, 1), 0.75), "sum")


def test_round_to_edges():
    """half to even, saturating, exact fp16 subnormals -- the rounding the kernels' cvt.rn.satfinite does."""
    assert Q.round_to(1 + 2.0 ** -11, "fp16") == 1.0 and Q.round_to(1 + 3 * 2.0 ** -11, "fp16") == 1 + 2.0 ** -9
    assert Q.round_to(70000.0, "fp16") == 65504.0 and Q.round_to(-1e9, "fp16") == -65504.0
    assert Q.round_to(3 * 2.0 ** -26, "fp16") == 2.0 ** -24 and Q.round_to(2.0 ** -26, "fp16") == 0.0
    assert Q.round_to(1 + 2.0 ** -8, "bf16") == 1.0 and Q.round_to(1 + 3 * 2.0 ** -8, "bf16") == 1 + 2.0 ** -6


# ---- every seeded fault breaks the exact comparison ---------------------------------------------------------------------
def _trunc16(x, fmt):
    """Truncation toward zero instead of round-to-nearest-even."""
    t, emin, _ = FORMATS[fmt]
    x = np.asarray(x, np.float64)
    q = ulp16(x, fmt)
    return np.trunc(x / q) * q


@pytest.mark.parametrize("fmt", FMTS)
def test_seeded_gemm_faults(fmt):
    rng = np.random.default_rng(4)
    M, K, N = 257, 320, 256
    a, w, b = dyadic(rng, (M, K)), dyadic(rng, (K, N)), dyadic(rng, (N,))
    ref = R.gemm_fwd(a, w, b, "relu", 0.25, fmt)[0]
    # a dropped last 64-deep k-block
    assert not _same(R.gemm_fwd(a[:, :K - 64], w[:K - 64], b, "relu", 0.25, fmt)[0], ref)
    # the bias added after the activation
    assert not _same(Q.round_to(np.maximum(a @ w, 0) + b, fmt), ref)
    # truncation instead of RN-even (operands on a 1/256 grid, so that fp16 rounds too)
    af = dyadic(rng, (M, K), k=255, den=256)
    assert not _same(_trunc16(np.maximum(af @ w + b, 0), fmt), R.gemm_fwd(af, w, b, "relu", 0.25, fmt)[0])
    # inf instead of saturation
    big = R.gemm_fwd(a * 64, w * 64, b, "linear", 0.25, "fp16")[0]
    assert not _same(Q.round_to(a * 64 @ (w * 64) + b, "fp16", saturate=False), big)
    # DGRAD: column sums of the rounded values; DGRAD without act'
    dz, x = dyadic(rng, (M, N)), rng.integers(-15, 16, size=(M, K)) / 16
    v = R.dgrad_values(dz, w, x, "tanh", 0.2)
    out, cs = R.gemm_dgrad(dz, w, x, "tanh", 0.2, fmt)
    assert not _same(R.dgrad_colsums(Q.round_to(v.astype(np.float64), fmt).astype(np.float32)), cs)
    assert not _same(Q.round_to(dz @ w.T, fmt), out)
    # WGRAD: 32-row slices whose 64-row k-block reads into the neighbour
    parts = R.gemm_wgrad(a, dz, M, -(-M // 32), 32, 1.0)
    leaky = np.stack([a[s * 32:min(M, s * 32 + 64)].T @ dz[s * 32:min(M, s * 32 + 64)] for s in range(-(-M // 32))])
    assert not _same(leaky, parts)


@pytest.mark.parametrize("fmt", FMTS)
def test_seeded_head_faults(fmt):
    rng = np.random.default_rng(5)
    n, out, nb = 1000, 3, 3
    g = np.maximum(dyadic(rng, (n, 256), k=2, den=2), 0)
    Wc, bc = dyadic(rng, (256, out), k=1, den=8), dyadic(rng, (out,), k=4, den=16)
    y = g @ Wc + bc + dyadic(rng, (n, out), k=2, den=16)
    ib, S = 2.0 ** -10, 2.0 ** 10
    ref = R.head(g, Wc, bc, "linear", "relu", 0.2, "mse", y, ib, S, nblocks=nb, fmt=fmt, z_kernel=g @ Wc + bc)
    # a row credited to the wrong block: the generic kernel's ROWS = 1 assignment with ROWS = 4 instead
    wrong = R.head_block_of_rows(n, nb, 2, False)
    assert not np.array_equal(wrong, R.head_block_of_rows(n, nb, out, False))
    dz = 2 * (g @ Wc + bc - y) / out * ib
    shifted = np.stack([(g[wrong == b].T @ dz[wrong == b]).ravel() for b in range(nb)])
    assert np.abs(shifted - ref["wpart"][:, :256 * out]).max() > (ref["wpart_bound"][:, :256 * out]).max()
    # the last hidden layer's dg without act' or without the loss scale
    d = S * (dz @ Wc.T) * (g > 0)
    assert np.all(np.abs(Q.round_to(d, fmt) - ref["dg"]) <= ref["dg_bound"])
    assert np.any(np.abs(Q.round_to(S * (dz @ Wc.T), fmt) - ref["dg"]) > ref["dg_bound"])
    assert np.any(np.abs(Q.round_to(dz @ Wc.T * (g > 0), fmt) - ref["dg"]) > ref["dg_bound"])


@pytest.mark.parametrize("fmt", FMTS)
def test_seeded_tail_faults(fmt):
    """K0 = 320: d emb leaves in 128-column chunks at c0 = 0, 128, 256, the last one half full (64 live columns).  Written
    chunk by chunk as e3 writes them, d emb equals the reference; each fault of one chunk breaks the exact comparison: the
    second chunk at the first chunk's offset, the half-full last chunk 64 columns early, only its first 32 columns written,
    or its W0 rows read 64 rows off.  dg2 without act' or without the loss scale is caught too."""
    a, W0, b0, W1, b1, wout, bout = _layers(6, M=300, K0=320)
    z = R.fwd2(a, W0, b0, W1, b1, wout, bout, "relu", 0.25, None, 1.0, 1.0, 4, fmt, stages=1)["z"]
    y = z[:, None] + 0.0625
    ref = R.fwd2(a, W0, b0, W1, b1, wout, bout, "relu", 0.25, y, 2.0 ** -9, 2.0 ** 9, 4, fmt, stages=3, demb=True)
    K0 = W0.shape[0]

    def chunked(fault=None):
        out = np.full(ref["demb"].shape, -1.0)                              # -1: never a d emb value here (the sentinel)
        for cc, c0 in enumerate(range(0, K0, 128)):
            width = min(128, K0 - c0)
            rows = np.arange(c0, c0 + width)
            if fault == "rows" and cc == 2:
                rows = rows - 64
            v = Q.round_to(ref["dg1"] @ W0[rows].T, fmt)
            dst = c0
            if fault == "offset" and cc == 1:
                dst = 0
            if fault == "early" and cc == 2:
                dst = c0 - 64
            if fault == "half" and cc == 2:
                width = 32
            out[:, dst:dst + width] = v[:, :width]
        return out

    assert _same(chunked(), ref["demb"])
    for fault in ("offset", "early", "half", "rows"):
        assert not _same(chunked(fault), ref["demb"]), fault
    g2 = Q.round_to(np.maximum(Q.round_to(np.maximum(a @ W0 + b0, 0), fmt) @ W1 + b1, 0), fmt)
    ds = 2 * (z - y[:, 0]) * 2.0 ** -9 * 2.0 ** 9
    assert _same(Q.round_to(ds[:, None] * wout * (g2 > 0), fmt), ref["dg2"])
    assert not _same(Q.round_to(ds[:, None] * wout, fmt), ref["dg2"])
    assert not _same(Q.round_to(ds[:, None] * wout * (g2 > 0) * 2.0 ** -9, fmt), ref["dg2"])


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act", ["tanh", "sigmoid", "elu"])
def test_sfu_tail_bounds(fmt, act):
    """The bounded tail reference (tanh / sigmoid / elu): a kernel that computes every stage in float64 and rounds where the
    kernel rounds lies inside every bound, continuing from its own stored g1, z, dg2 and dg1; dg2 without act' or a
    tile's dg1 column sums dropped leave them."""
    a, W0, b0, W1, b1, wout, bout = _layers(7, M=300, K0=320)
    rng = np.random.default_rng(8)
    y = dyadic(rng, (300, 1))
    ib, S = 2.0 ** -9, 2.0 ** 9
    d0 = a @ W0 + b0
    act_f = {"tanh": np.tanh, "sigmoid": lambda v: 1 / (1 + np.exp(-v)), "elu": lambda v: np.where(v > 0, v, np.expm1(np.minimum(v, 0)))}[act]
    g1 = Q.round_to(act_f(d0), fmt)
    g2 = Q.round_to(act_f(g1 @ W1 + b1), fmt)
    z = g2 @ wout + bout[0]
    ds = 2 * (z - y[:, 0]) * ib * S
    ap = {"tanh": 1 - g2 * g2, "sigmoid": g2 * (1 - g2), "elu": np.where(g2 > 0, 1.0, g2 + 1)}[act]
    dg2 = Q.round_to(ds[:, None] * wout * ap, fmt)
    a1 = {"tanh": 1 - g1 * g1, "sigmoid": g1 * (1 - g1), "elu": np.where(g1 > 0, 1.0, g1 + 1)}[act]
    v1 = (dg2 @ W1.T) * a1
    dg1 = Q.round_to(v1, fmt)
    kern = dict(g1=g1, z=z, dg2=dg2, dg1=dg1)
    ref = R.fwd2_sfu(a, W0, b0, W1, b1, wout, bout, act, 0.2, y, ib, S, 2, fmt, kern, stages=3, demb=True)
    within = lambda got, key: np.all(np.abs(got - ref[key]) <= ref[key + "_bound"])
    assert within(g1, "g1") and within(z, "z") and within(dg2, "dg2") and within(dg1, "dg1")
    assert within(Q.round_to(dg1 @ W0.T, fmt), "demb")
    assert within(np.stack([v1[:128].sum(0), v1[128:256].sum(0), v1[256:].sum(0)]), "dbpart")
    assert not within(Q.round_to(ds[:, None] * wout, fmt), "dg2")
    assert not within(np.stack([v1[:128].sum(0), v1[128:256].sum(0), 0 * v1[256:].sum(0)]), "dbpart")
