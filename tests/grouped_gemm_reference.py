"""TEST INFRASTRUCTURE ONLY -- the float64 reference of the grouped dense-layer GEMM kernels (dib_gemm_simt.cu, exact fp32
FMA, and dib_gemm_tc.cu, tf32 wgmma) on exact operands: every A / B / bias entry on the grid 1/4, every DGRAD activation
source on the grid 1/16, so that with reductions of at most 512 terms every sum the kernels form is exact (asserted with
``fp_exact.fits``, in units of the grid) and the kernels must equal this bit for bit.  It rounds only where the kernels
round: one fp32 rounding of alpha * z (leaky ReLU FWD) and of o * act'(x) (DGRAD), and cvt.rna.tf32 under round_out.
tanh / sigmoid / elu in FWD (libdevice) are the one inexact case, returned in float64 and held to a ulp bound by the GPU
test.  Not collected by pytest (no test_ prefix)."""
import numpy as np

from oracle import dib_oracle as O
from tests.fp_exact import act_grad32, fits, round_tf32

INEXACT_ACTS = ("tanh", "sigmoid", "elu")


def act_source(rng, shape):
    """DGRAD activation sources k / 16 in (-1, 1), exact zeros included."""
    return (rng.integers(-15, 16, size=shape) / 16).astype(np.float32)


def assert_on_grid(a, den):
    a = np.asarray(a, np.float64)
    assert np.array_equal(a * den, np.round(a * den)), f"operand off the 1/{den} grid"


def act_fwd32(act, z, alpha):
    """The FWD epilogue act(z) on the exact fp32 z; leaky ReLU rounds alpha * z once in fp32.  Inexact activations are
    returned in float64 (compared with a ulp bound)."""
    if act == "linear":
        return z
    if act == "relu":
        return np.maximum(z, 0.0)
    if act == "leaky_relu":
        z32 = z.astype(np.float32)
        return np.where(z32 > 0, z32, np.float32(alpha) * z32).astype(np.float64)
    return O.act_fwd(act, z)


def ref_fwd(a, w, b, act, alpha, round_out):
    """act(a w + b) of one problem: a [M x T], w [T x C], b [C]."""
    for v in (a, w, b):
        assert_on_grid(v, 4)
    fits((np.abs(a.astype(np.float64)) @ np.abs(w.astype(np.float64)) + np.abs(b)) * 16, 1.0, "FWD sums")
    z = a.astype(np.float64) @ w.astype(np.float64) + b.astype(np.float64)
    out = act_fwd32(act, z, alpha)
    if act in INEXACT_ACTS:
        return out
    out32 = out.astype(np.float32)
    assert np.array_equal(out32.astype(np.float64), out)
    return round_tf32(out32) if round_out else out32


def ref_dgrad(dz, w, x, act, alpha, round_out):
    """(dz w^T) * act'(x) of one problem: dz [M x T], w [C x T] (the layer's [fan-in x fan-out] kernel), x [M x C]."""
    for v in (dz, w):
        assert_on_grid(v, 4)
    o = dz.astype(np.float64) @ w.astype(np.float64).T
    bound = np.abs(dz.astype(np.float64)) @ np.abs(w.astype(np.float64)).T * 16
    if act == "linear":
        fits(bound, 1.0, "DGRAD sums")
        out = o.astype(np.float32)
    else:
        assert_on_grid(x, 16)
        g = act_grad32(act, x, alpha)
        if not (act == "leaky_relu" and np.float32(alpha) * 4 != np.round(np.float32(alpha) * 4)):
            assert_on_grid(g, 256)
            fits(bound * 256, 1.0, "DGRAD o * act'")
        out = o.astype(np.float32) * g               # one fp32 rounding (exact unless alpha is off the grid)
    return round_tf32(out) if round_out else out


def ref_wgrad(h, dz, M, nsplit, rps):
    """Per-split partials of h^T dz and of the column sums of dz over batch rows [s rps, min(M, (s + 1) rps))."""
    for v in (h, dz):
        assert_on_grid(v, 4)
    R, C = h.shape[1], dz.shape[1]
    dw, db = np.zeros((nsplit, R, C), np.float32), np.zeros((nsplit, C), np.float32)
    for s in range(nsplit):
        lo, hi = s * rps, min(M, (s + 1) * rps)
        if hi <= lo:
            continue
        hs, ds = h[lo:hi].astype(np.float64), dz[lo:hi].astype(np.float64)
        fits(np.abs(hs).T @ np.abs(ds) * 16, 1.0, "WGRAD sums")
        fits(np.abs(ds).sum(0) * 4, 1.0, "bias column sums")
        dw[s] = (hs.T @ ds).astype(np.float32)
        db[s] = ds.sum(0).astype(np.float32)
    return dw, db


def ulp32(x):
    """fp32 unit in the last place of |x| (the spacing above it)."""
    x = np.abs(np.asarray(x, np.float32))
    return (np.nextafter(x, np.float32(np.inf)) - x).astype(np.float64)
