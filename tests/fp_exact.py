"""TEST INFRASTRUCTURE ONLY -- the floating-point model the kernel references share: the unit roundoff and gamma_m of the
running error analysis, fp32 / tf32 / 16-bit rounding, the exact-operand tools (dyadic grids and the 24-bit fit), the
activation derivatives as the kernels form them, and the per-element bound checker.  Not collected by pytest (no test_
prefix).  numpy only; it imports nothing else from tests/."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24               # fp32 unit roundoff
C_BOUND = 2.0                # reported bound = C_BOUND x the first-order error: covers every product of two or more errors
TINY = 2.0 ** -126           # the smallest normal fp32 value
EXACT_BITS = 24              # fp32 significand bits: sums of integer multiples of a unit below 2^24 units are exact

# significand bits t (incl. the implicit one), minimum normal exponent, largest finite value
FORMATS = {
    "fp16": (11, -14, 65504.0),
    "bf16": (8, -126, (2.0 - 2.0 ** -7) * 2.0 ** 127),
}


def gamma(m):
    m = np.asarray(m, np.float64)
    return m * U / (1.0 - m * U)


# ---- fp32 / tf32 ----------------------------------------------------------------------------------------------------------
def f32(x):
    """x rounded to fp32, as a float32 array"""
    return np.asarray(x, np.float64).astype(np.float32)


def is_fp32(x):
    """elementwise: x is an fp32 value"""
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64) == x


def round_tf32(x):
    """cvt.rna.tf32.f32: round the fp32 value to 10 explicit mantissa bits, to nearest, ties away from zero, as a float32
    array.  On the bit pattern of a finite value that is adding half of the dropped unit to the magnitude bits and clearing
    the low 13 bits (a carry moves into the exponent); NaN and inf pass unchanged."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32)
    r = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return np.where(np.isfinite(x), r, u).astype(np.uint32).view(np.float32)


# ---- 16-bit formats -------------------------------------------------------------------------------------------------------
def round_to(x, fmt, saturate=True):
    """Round half to even to the 16-bit format ``fmt`` ('fp16' | 'bf16' | None = no rounding), in float64.  Subnormals are
    exact (the quantum never drops below 2^(emin - t + 1)).  ``saturate``: a result beyond the largest finite value becomes
    +-max (cvt.rn.satfinite; infinities too), else +-inf (cvt.rn / __float2half_rn).  NaN stays NaN."""
    x = np.asarray(x, dtype=np.float64)
    if fmt is None:
        return x
    t, emin, vmax = FORMATS[fmt]
    finite = np.isfinite(x)
    xf = np.where(finite, x, 0.0)
    _, ex = np.frexp(xf)                                    # |x| = m 2^ex, m in [0.5, 1): leading bit 2^(ex - 1)
    e = np.maximum(ex - 1, emin)
    q = np.ldexp(1.0, e - (t - 1))                          # the quantum (ulp) at that exponent
    r = np.round(xf / q) * q                                # x / q is exact (power-of-two scaling); np.round: half to even
    if saturate:
        r = np.clip(r, -vmax, vmax)
        r = np.where(np.isinf(x), np.sign(x) * vmax, r)
    else:
        r = np.where(np.abs(r) > vmax, np.copysign(np.inf, r), r)
        r = np.where(np.isinf(x), x, r)
    return np.where(np.isnan(x), np.nan, r)


def r16(x, fmt):
    return round_to(x, fmt)


def ulp16(x, fmt):
    """The 16-bit ulp at |x| (the quantum of round_to)."""
    t, emin, _ = FORMATS[fmt]
    _, ex = np.frexp(np.abs(np.asarray(x, np.float64)))
    return np.ldexp(1.0, np.maximum(ex - 1, emin) - (t - 1))


def to16(v, fmt):
    """16-bit bit patterns (int16) of float64 values representable in fmt."""
    v = np.asarray(v, np.float64)
    if fmt == "fp16":
        h = v.astype(np.float16)
        assert np.array_equal(h.astype(np.float64), v, equal_nan=True), "value not representable in fp16"
        return h.view(np.int16)
    f = v.astype(np.float32)
    u = f.view(np.uint32)
    assert np.array_equal(f.astype(np.float64), v, equal_nan=True) and not np.any(u & 0xFFFF), "value not representable in bf16"
    return (u >> 16).astype(np.uint16).view(np.int16)


def from16(b, fmt):
    b = np.asarray(b).view(np.int16)
    if fmt == "fp16":
        return b.view(np.float16).astype(np.float64)
    return (b.view(np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


# ---- exact operands and the 24-bit fit ------------------------------------------------------------------------------------
def dyadic(rng, shape, k=4, den=4, dtype=np.float64):
    """Operands on the grid i / den, |i| <= k (exact in fp16, bf16 and tf32 for den <= 2^7 and k <= 2^8)."""
    return (rng.integers(-k, k + 1, size=shape) / den).astype(dtype)


def sparse_dyadic(rng, shape, k=4, den=4, density=0.25):
    v = dyadic(rng, shape, k, den)
    return np.where(rng.random(shape) < density, v, 0.0)


def quantum(a):
    """The smallest power of two every entry of ``a`` is a multiple of (1 for an all-zero array)."""
    a = np.abs(np.asarray(a, np.float64)).ravel()
    a = a[a > 0]
    if a.size == 0:
        return 1.0
    m, e = np.frexp(a)                                                  # a = m 2^e, m in [0.5, 1)
    mi = (m * 2.0 ** 53).astype(np.int64)                               # an integer: a = mi 2^(e - 53)
    low = np.frexp((mi & -mi).astype(np.float64))[1] - 1               # its lowest set bit
    return float(np.ldexp(1.0, int((e - 53 + low).min())))


def fits(term_abs_sum, unit, what):
    """Every value a kernel forms from terms whose magnitudes sum to ``term_abs_sum`` is an integer multiple of ``unit``
    below 2^24 units: exact in fp32 in any order."""
    m = float(np.max(np.asarray(term_abs_sum, np.float64), initial=0.0)) / unit
    assert m < 2.0 ** EXACT_BITS, f"{what}: {m:.4g} units need more than {EXACT_BITS} bits"


def exact_matmul(a, b, what):
    """a @ b in float64, asserting that fp32 forms it exactly in any order."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fits(np.abs(a) @ np.abs(b), quantum(a) * quantum(b), what)
    return a @ b


# ---- activation derivatives from the output h (dib_act_grad) --------------------------------------------------------------
def act_grad(act, h, alpha):
    """act'(h) in float64 and the error bound of its fp32 evaluation (sigmoid h (1 - h): two roundings, 2u |h (1 - h)|)"""
    h = np.asarray(h, np.float64)
    if act == "relu":
        return (h > 0).astype(np.float64), np.zeros_like(h)
    if act == "leaky_relu":
        return np.where(h > 0, 1.0, float(np.float32(alpha))), np.zeros_like(h)
    if act == "tanh":
        v = 1.0 - h * h
        return v, U * h * h + U * np.abs(v)
    if act == "sigmoid":
        v = h * (1.0 - h)
        return v, 2 * U * np.abs(v)
    if act == "elu":
        return np.where(h > 0, 1.0, h + 1.0), np.where(h > 0, 0.0, U * np.abs(h + 1.0))
    return np.ones_like(h), np.zeros_like(h)


def act_grad32(act, h, alpha):
    """act'(h) in fp32 (float32 array) as the kernels form it; exact for h on the 1/16 grid."""
    h = f32(h)
    one = np.float32(1)
    if act == "relu":
        return (h > 0).astype(np.float32)
    if act == "tanh":
        return one - h * h
    if act == "leaky_relu":
        return np.where(h > 0, one, np.float32(alpha)).astype(np.float32)
    if act == "sigmoid":
        return h * (one - h)
    if act == "elu":
        return np.where(h > 0, one, h + one).astype(np.float32)
    return np.ones_like(h)


# ---- the per-element bound checker ------------------------------------------------------------------------------------------
def within(worst, what, got, ref, bound, tag):
    """|got - ref| <= bound everywhere (a NaN anywhere fails); prints and records in ``worst`` (the calling suite's table,
    keyed by ``what``) the largest measured / bound over the elements with a non-zero bound."""
    got, ref, bound = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.asarray(bound, np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{tag} {what}: {bad.sum()} of {bad.size} elements outside their bound; first at "
                           f"{np.argwhere(bad)[0].tolist()}: got {got[bad][0]!r} ref {ref[bad][0]!r} bound {bound[bad][0]!r}")
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    worst[what] = max(worst.get(what, 0.0), ratio)
    print(f"{tag} {what}: worst measured / bound {ratio:.3g}; exact elements {int((~pos).sum())}")


def within_same_nans(worst, what, got, ref, bound, tag):
    """``within`` on the elements where ref is a number, after asserting that got is NaN exactly where ref is"""
    got, ref, bound = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.asarray(bound, np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{tag} {what}: NaN where the reference has none, or the reverse"
    within(worst, what, got[~nan], ref[~nan], bound[~nan], tag)
