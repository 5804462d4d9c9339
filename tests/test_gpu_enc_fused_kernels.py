"""GPU (H100): the fused encoder kernels of dib_enc_fused.cu -- the weight pack, dib_enc_fused_fwd_kernel and
dib_enc_fused_bwd_kernel, both instantiations of each (relu / the other activations) -- launched through
dib_debug_enc_fused exactly as the step launches them, on chosen grids, against tests/enc_fused_reference.py in fp16 and
bf16.

Exact cases (relu, leaky ReLU with alpha = 1/4 and linear; dyadic x, weights, eps and d emb; lv = 0) must match the float64
reference bit for bit in every output element: the packed image, emb (TF32), user_emb, emb16, the KL table and every
weight-gradient partial.  The one exception is the sign of an exact zero that the tensor core fixes (a sum of products
that cancels, an accumulator that a zero operand leaves at +-0): the reference cannot restate it, so zeros compare by value.

Bounded cases print their worst measured / bound ratio (WORST): the positional encoding read out through the first-layer
operand against r(sin(f x)) within enc_fused_reference.SIN_TOL, and the Philox noise against oracle/philox within
Z_TOL (1 + |z|).

Memory contracts, in every call: NaN in every input element the kernels must not read (other x columns and rows past n,
eps and d emb of rows past n and pad columns, parameter gaps), a sentinel in every element they must not write (emb rows
past n and pad columns, slot rows a feature does not own, the partial table's gaps), and one launch per phase."""
import ctypes

import numpy as np
import pytest
import torch

from tests import enc_fused_reference as R
from tests.fused16_oracle import loss_scale
from tests.fp_exact import dyadic, from16, r16, to16, ulp16
from tests.gpu_cases import _L, _sms

pytestmark = pytest.mark.gpu

ACT = {a: i for i, a in enumerate(R.ACTS)}
FMTS = ["fp16", "bf16"]
NAN16 = {"fp16": 0x7E00, "bf16": 0x7FC0}
SENT16 = np.int16(-8531)                 # 0xDEAD: finite in both formats, never a result here
SENT32 = np.float32(-7777.25)
WORST = {}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def same(got, want, what, zeros_by_value=False, bits=None):
    """got / want float64 arrays of one output; the bit patterns (bits: the converter of a value array) of every element
    must agree.  zeros_by_value: an exact zero matches a zero of either sign -- only for the weight-gradient partials,
    whose zeros are tensor-core sums (of products that cancel, or of zero products) with a sign the reference cannot
    restate.  u = fma(sv, eps, mu) is +0 whenever it is zero (eps is never -0 here), and the KL sums start from +0, so
    emb, user_emb, emb16 and the KL table compare bit for bit."""
    bits = bits or (lambda v: np.asarray(v, np.float32).view(np.uint32))
    eq = bits(got) == bits(want)
    if zeros_by_value:
        eq |= (got == 0) & (want == 0)
    if not eq.all():
        bad = np.argwhere(~eq)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} elements differ, first at {i}: got {got[i]!r}, want {want[i]!r}")


def bits16(fmt):
    return lambda v: to16(v, fmt)


# ---------------------------------------------------------------------------------------------------------------------
# one call of the hook
# ---------------------------------------------------------------------------------------------------------------------
class Case:
    """Inputs of one call: fdims, nfreq, activation, n, the parameters (R.pack's input), x and the layout tables."""

    def __init__(self, fmt, fdims, nfreq, act, n, enc, x_cols, x_off, ldx, logvar_offset=0.0, alpha=0.25, gap=3):
        self.fmt, self.fdims, self.nfreq, self.act, self.n, self.enc = fmt, tuple(fdims), nfreq, act, n, enc
        self.F = len(fdims)
        self.alpha, self.logvar_offset = alpha, logvar_offset
        self.lay, self.count = R.layout(fdims, nfreq, gap)
        self.params = R.flatten_params(enc, self.lay, self.count).astype(np.float32)
        in_block = np.zeros(self.count, bool)
        for b in R.BLOCKS:
            for f in range(self.F):
                size = {"w0": fdims[f] * nfreq * R.HID, "b0": R.HID, "w1": R.HID * R.HID, "b1": R.HID, "w2": R.HID * R.EO,
                        "b2": R.EO}[b]
                in_block[int(self.lay[b][f]):int(self.lay[b][f]) + size] = True
        self.params[~in_block] = np.nan
        self.x_off, self.ldx = np.asarray(x_off, np.int32), ldx
        self.x = np.full((n + 3, ldx), np.nan, np.float32)
        for f, d in enumerate(fdims):
            self.x[:n, x_off[f]:x_off[f] + d] = x_cols[f]
        self.img = R.pack(enc, fdims, nfreq, logvar_offset, fmt)


def make_case(fmt, fdims, nfreq, act, n, seed=0, logvar_offset=-3.0, x_gap=1, density=1 / 16, x=None, enc=None, alpha=0.25):
    rng = np.random.default_rng(seed)
    enc = enc if enc is not None else R.exact_params(rng, fdims, nfreq, logvar_offset, density)
    x_off, pos = [], 1
    for d in fdims:
        x_off.append(pos)
        pos += d + x_gap
    ldx = pos + 1 if pos % 2 == 0 else pos                                  # odd
    cols = [x[f] if x is not None else dyadic(rng, (n, d), 4, 2) for f, d in enumerate(fdims)]
    return Case(fmt, fdims, nfreq, act, n, enc, cols, x_off, ldx, logvar_offset, alpha)


def run(c, phases=7, grid=0, eps=None, d_emb=None, d_emb16=None, beta=0.75, inv_batch=None, S=None, seed=11, step=5,
        step_dev=None, sample_offset=0, over=None):
    """Runs the hook and returns its outputs (host arrays).  eps [n, F, 32] or None (Philox).  over: hook arguments by name
    that replace the ones run() forms (the refusal tests)."""
    L = _L()
    lib = L.load()
    F, n = c.F, c.n
    E = R.E
    tiles = -(-n // R.TM)
    if grid == 0:
        g_fwd, g_bwd = min(F * tiles, 2 * _sms()), min(F * tiles, _sms())
    else:
        g_fwd = g_bwd = grid
    slots = -(-max(g_fwd, g_bwd) // F)
    kl_stride = slots + 1
    ld = F * E + 2
    ld16 = F * E + 8
    t = {}
    t["params"] = dev(c.params)
    t["x"] = dev(c.x)
    if eps is not None:
        e = np.full((n + 3, F, E), np.nan, np.float32)
        e[:n] = eps
        t["eps"] = dev(e)
    t["emb"] = dev(np.full((n + 3, ld), SENT32, np.float32))
    t["user"] = dev(np.full((n + 3, F * E), SENT32, np.float32))
    t["emb16"] = dev(np.full((n + 3, ld), SENT16, np.int16))
    t["kl"] = dev(np.full((F, kl_stride), SENT32, np.float32))
    t["packed"] = dev(np.zeros(F * R.PACK_ELEMS, np.int16)) if phases & 1 else dev(to16(c.img, c.fmt).ravel())
    split_stride = c.count + 64 + (c.count % 2)
    t["part"] = dev(np.full((slots + 1, split_stride), SENT32, np.float32))
    if d_emb is not None:
        g = np.full((n + 3, ld), np.nan, np.float32)
        g[:n, :F * E] = d_emb
        t["d_emb"] = dev(g)
    if d_emb16 is not None:
        g = np.full((n + 3, ld16), np.int16(np.uint16(NAN16[c.fmt]).view(np.int16)), np.int16)
        g[:n, :F * E] = to16(d_emb16, c.fmt)
        t["d_emb16"] = dev(g)
    t["beta"] = dev(np.array([beta], np.float32))
    if step_dev is not None:
        t["step_dev"] = dev(np.array([step_dev], np.uint32).view(np.int32))
    S = S if S is not None else loss_scale(n)
    inv_batch = inv_batch if inv_batch is not None else 1.0 / n
    p = lambda k: L.ptr(t[k]) if k in t else None
    keep = [(ctypes.c_int64 * F)(*[int(v) for v in c.lay[b]]) for b in R.BLOCKS]
    keep += [(ctypes.c_int32 * F)(*c.fdims), (ctypes.c_int32 * F)(*[int(v) for v in c.x_off])]
    tabs = dict(zip(R.BLOCKS, (ctypes.cast(a, ctypes.c_void_p) for a in keep)))
    fd, xo = (ctypes.cast(a, ctypes.c_void_p) for a in keep[6:])
    before = int(lib.dib_launch_count())
    args = dict(phases=phases, F=F, fdim=fd, x_off=xo, nfreq=c.nfreq, act=ACT[c.act], alpha=c.alpha,
                bf16=1 if c.fmt == "bf16" else 0, logvar_offset=c.logvar_offset, params=p("params"), param_count=c.count,
                w0_off=tabs["w0"], b0_off=tabs["b0"], w1_off=tabs["w1"], b1_off=tabs["b1"], w2_off=tabs["w2"],
                b2_off=tabs["b2"], grid=grid, n=n, x=p("x"), ldx=c.ldx, eps=p("eps"), seed=seed, step=step,
                step_dev=p("step_dev"), sample_offset=sample_offset, emb=p("emb"), ldemb=ld, user_emb=p("user"),
                emb16=p("emb16"), ldemb16=ld, kl_part=p("kl"), kl_stride=kl_stride, d_emb=p("d_emb"), ldd=ld,
                d_emb16=p("d_emb16"), ldd16=ld16, beta_dev=p("beta"), inv_batch=inv_batch, gscale=S, part=p("part"),
                split_stride=split_stride, packed=p("packed"), stream=ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    for k, v in (over or {}).items():
        assert k in args, k
        args[k] = v(args[k]) if callable(v) else v
    rc = lib.dib_debug_enc_fused(*args.values())
    assert rc == 0, lib.dib_last_error().decode()
    launches = int(lib.dib_launch_count()) - before
    assert launches == bin(phases & 7).count("1"), launches
    out = {k: host(v) for k, v in t.items()}
    out.update(g_fwd=g_fwd, g_bwd=g_bwd, slots=slots, kl_stride=kl_stride, split_stride=split_stride, S=S,
               inv_batch=inv_batch, ld=ld)
    return out


def check_forward(c, out, eps, what):
    """emb, user_emb, emb16 and the KL table of the exact regime, plus the sentinels around them."""
    F, n, E, ld = c.F, c.n, R.E, out["ld"]
    ref = R.forward(c.img, c.x, c.x_off, c.fdims, c.nfreq, c.act, c.alpha, c.fmt, n, eps, out["g_fwd"])
    emb, user, e16 = out["emb"], out["user"], out["emb16"]
    assert np.all(emb[n:] == SENT32) and np.all(emb[:, F * E:] == SENT32), f"{what}: emb written outside rows < n x 32 F"
    assert np.all(user[n:] == SENT32), f"{what}: user_emb written past n"
    assert np.all(e16[n:] == SENT16) and np.all(e16[:, F * E:] == SENT16), f"{what}: emb16 written outside"
    same(emb[:n, :F * E].astype(np.float64), ref["emb"], what + " emb")
    same(user[:n].astype(np.float64), ref["user_emb"], what + " user_emb")
    same(from16(e16[:n, :F * E], c.fmt), ref["emb16"], what + " emb16", bits=bits16(c.fmt))
    kl = out["kl"].astype(np.float64)
    want = np.zeros_like(kl)                                            # cleared by the pack phase
    want[:, :ref["kl_part"].shape[1]] = ref["kl_part"]
    same(kl, want, what + " kl_part")
    return ref


def check_backward(c, out, ref_fw, eps, g, beta, what):
    parts = R.backward(c.img, ref_fw["chains"], c.fdims, c.nfreq, c.act, c.alpha, c.fmt, c.n, eps, g, beta, out["inv_batch"],
                       out["S"], out["g_bwd"], c.lay)
    want = R.partial_table(parts, c.lay, out["split_stride"], out["slots"] + 1, float(SENT32))
    same(out["part"].astype(np.float64), want, what + " partials", zeros_by_value=True)


def check_pack(c, out):
    same(from16(out["packed"].reshape(c.F, R.PACK_ELEMS), c.fmt), c.img, "packed image", bits=bits16(c.fmt))


def exact_inputs(c, seed=1, gscale_rows=None):
    rng = np.random.default_rng(seed)
    eps = dyadic(rng, (c.n, c.F, R.E), 4, 2)
    S = loss_scale(gscale_rows or c.n)
    d_emb = (dyadic(rng, (c.n, c.F * R.E), 4, 4) / S).astype(np.float32)
    return eps, d_emb, S


def full_exact(fmt, act, fdims, nfreq, n, grid, route="fp32", beta=0.75, seed=0, density=1 / 16, inv_batch=None,
               d_scale=1.0):
    c = make_case(fmt, fdims, nfreq, act, n, seed=seed, density=density)
    eps, d_emb, S = exact_inputs(c, seed + 1)
    d_emb = (d_emb * np.float32(d_scale)).astype(np.float32)
    g = (d_emb.astype(np.float32) * np.float32(S)).astype(np.float64)
    kw = dict(d_emb=d_emb) if route == "fp32" else dict(d_emb16=g)
    # 1 / S as inv_batch keeps bs = beta inv_batch S on the operands' grid (1 / n would not be a power of two)
    out = run(c, 7, grid, eps=eps, beta=beta, S=S, inv_batch=inv_batch or 1.0 / S, **kw)
    what = f"{fmt} {act} fdims={fdims} nfreq={nfreq} n={n} grid={grid} {route}"
    check_pack(c, out)
    ref = check_forward(c, out, eps, what)
    check_backward(c, out, ref, eps, g, beta, what)


# ---------------------------------------------------------------------------------------------------------------------
# exact cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["relu", "linear", "leaky_relu"])
@pytest.mark.parametrize("fmt", FMTS)
def test_both_instantiations_mixed_fdims(fmt, act):
    n = 300 if act != "leaky_relu" else 200
    full_exact(fmt, act, (1, 3, 2), 1, n, 0, density=1 / 16 if act != "leaky_relu" else 1 / 64)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, 128 * 5 + 77])
@pytest.mark.parametrize("fmt", FMTS)
def test_batch_edges(fmt, n):
    full_exact(fmt, "relu", (2, 1), 1, n, 0)


@pytest.mark.parametrize("route", ["fp32", "d16"])
@pytest.mark.parametrize("fmt", FMTS)
def test_one_slot_sums_many_tiles(fmt, route):
    full_exact(fmt, "relu", (1,), 1, 128 * 20 + 5, 1, route=route)


@pytest.mark.parametrize("F", [1, 3, 5, 16])
def test_every_schedule(F):
    n = 300
    tiles = 3
    fdims = tuple(1 + (f % 3) for f in range(F))
    for grid in sorted({1, 2, max(F - 1, 1), F, F + 1, 2 * F - 1, F * tiles, 0}):
        if grid > F * tiles:
            continue
        for fmt, route in (("fp16", "fp32"), ("bf16", "d16"), ("fp16", "d16")):
            full_exact(fmt, "relu" if grid % 3 else "linear", fdims, 1, n, grid, route=route)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("route", ["fp32", "d16"])
@pytest.mark.parametrize("beta", [0.0, 0.75])
@pytest.mark.parametrize("n", [1024, 1025])
def test_backward_routes_and_loss_scale(route, beta, n, fmt):
    full_exact(fmt, "relu", (1, 2), 1, n, 0, route=route, beta=beta)


@pytest.mark.parametrize("fmt", FMTS)
def test_subnormal_gradient_operands(fmt):
    """d emb S on the order of 2^-20: dO, dz2 and dz1 are fp16 subnormals (exact on the 2^-24 grid)."""
    full_exact(fmt, "relu", (1, 2), 1, 200, 0, beta=0.0, d_scale=2.0 ** -18)


@pytest.mark.parametrize("fmt", FMTS)
def test_pack_bias_carriers_offset_saturation(fmt):
    rng = np.random.default_rng(5)
    fdims, nfreq = (2, 1, 3), 5
    enc = R.exact_params(rng, fdims, nfreq, 0.0)
    for e in enc:                                                       # arbitrary fp32 values: every rounding of the pack
        for k in e:
            e[k] = rng.standard_normal(np.shape(e[k])).astype(np.float32).astype(np.float64)
    enc[0]["W1"][3, 5] = 1e5                                            # saturates in fp16
    enc[1]["b2"][40] = -1e5
    c = make_case(fmt, fdims, nfreq, "relu", 10, enc=enc, logvar_offset=-2.9)
    out = run(c, 1)
    check_pack(c, out)
    assert np.all(out["kl"] == 0), "the pack phase clears the KL table"
    if fmt == "fp16":
        assert 65504.0 in c.img[0] and -65504.0 in c.img[1]


# ---------------------------------------------------------------------------------------------------------------------
# the positional encoding, read out through the first-layer operand
# ---------------------------------------------------------------------------------------------------------------------
def pe_readout(fmt, act, fdims, nfreq, x_cols, n):
    c = make_case(fmt, fdims, nfreq, act, n, x=x_cols, enc=R.pe_readout_params(fdims, nfreq, act), logvar_offset=0.0)
    out = run(c, 3, 0, eps=np.zeros((n, c.F, R.E)))
    e16 = from16(out["emb16"][:n], fmt)
    assert np.all(out["emb16"][n:] == SENT16)
    res = []
    for f, d in enumerate(fdims):
        w_in = d * nfreq
        got = e16[:, f * R.E:f * R.E + w_in]
        assert np.all(e16[:, f * R.E + w_in] == 1.0), "the ones column must read 1 on every row inside the batch"
        assert np.all(e16[:, f * R.E + w_in + 1:(f + 1) * R.E] == 0.0)
        res.append((got, R.sin_values(x_cols[f], d, nfreq)))
    return res


LAYOUTS = [(1, 1), (3, 1), (1, 5), (2, 7), (3, 5), (1, 15)]


@pytest.mark.parametrize("act", ["relu", "linear"])
@pytest.mark.parametrize("fmt", FMTS)
def test_pe_operand_exact_where_the_sine_is_far_from_a_midpoint(fmt, act):
    """Every layout's [pe | 1] operand, read out bit for bit, at x whose sines lie farther than SIN_TOL from a midpoint."""
    rng = np.random.default_rng(9)
    for d, nfreq in LAYOUTS:
        n = 129
        xs = dyadic(rng, (4 * n, d), 256, 128)
        xs = xs[R.pe_exact(xs, d, nfreq, fmt)][:n]
        assert len(xs) == n
        for got, s in pe_readout(fmt, act, (d,), nfreq, [xs], n):
            same(got, r16(s, fmt), f"{fmt} {act} pe operand d={d} nfreq={nfreq}", bits=bits16(fmt))


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("layout,xmax", [((1, 5), 1000.0), ((3, 5), 1000.0), ((1, 15), 4.0), ((2, 7), 100.0)])
def test_pe_accuracy_at_large_arguments(fmt, layout, xmax):
    """r(dib_sin_pe(f x)) within SIN_TOL of sin(f x) before the 16-bit rounding, at |f x| up to 1.6e4 (nfreq 5, |x| 1e3)
    and 3.3e4 (nfreq 15, |x| 4)."""
    d, nfreq = layout
    rng = np.random.default_rng(10)
    n = 2000
    xs = rng.uniform(-xmax, xmax, (n, d)).astype(np.float32)
    (got, s), = pe_readout(fmt, "relu", (d,), nfreq, [xs], n)
    lo, hi = r16(s - R.SIN_TOL, fmt), r16(s + R.SIN_TOL, fmt)
    ok = (got >= lo) & (got <= hi)
    half = 0.5 * ulp16(s, fmt)
    ratio = np.maximum(np.abs(got - s) - half, 0.0) / R.SIN_TOL
    worst = float(ratio.max())
    WORST[f"pe {fmt} d={d} nfreq={nfreq} |x|<={xmax:g}"] = worst
    print(f"pe {fmt} d={d} nfreq={nfreq} |x| <= {xmax:g}: worst (|got - sin| - ulp/2) / SIN_TOL = {worst:.3g}")
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{int((~ok).sum())} operands outside SIN_TOL, first at {i}: x = {xs[i[0]]}, got {got[i]!r}, "
                             f"sin = {s[i]!r}")


# ---------------------------------------------------------------------------------------------------------------------
# the noise
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_philox_noise_readout(fmt):
    fdims, n = (1, 2, 1), 300
    c = make_case(fmt, fdims, 1, "relu", n, enc=R.noise_readout_params(np.random.default_rng(3), fdims, 1), logvar_offset=0.0)
    seed, step, sdev, off = 0x1234_5678_9ABC, 40, 7, 2 ** 32 + 12345
    out = run(c, 3, 0, seed=seed, step=step, step_dev=sdev, sample_offset=off)
    z = R.philox_noise(seed, step + sdev, off, n, c.F)
    got = out["user"][:n].astype(np.float64).reshape(n, c.F, R.E)
    err = np.abs(got - z) / (R.Z_TOL * (1 + np.abs(z)))
    WORST[f"noise {fmt}"] = float(err.max())
    print(f"noise {fmt}: worst |u - z| / (Z_TOL (1 + |z|)) = {err.max():.3g}")
    assert err.max() <= 1.0
    same(from16(out["emb16"][:n, :c.F * R.E], fmt), r16(got.reshape(n, -1), fmt), "emb16 = r(noise)", bits=bits16(fmt))
    # step + *step_dev is the summed step, bit for bit
    out2 = run(c, 3, 0, seed=seed, step=step + sdev, sample_offset=off)
    assert np.array_equal(out2["user"].view(np.uint32), out["user"].view(np.uint32))
    # the backward's noise is the forward's: Philox and eps = the forward's readout give identical partials
    ce = make_case(fmt, fdims, 1, "relu", n, seed=4)
    eps_dyad, d_emb, S = exact_inputs(ce, 5)
    b1 = run(ce, 5, 0, d_emb=d_emb, S=S, seed=seed, step=step, step_dev=sdev, sample_offset=off)
    b2 = run(ce, 5, 0, eps=got, d_emb=d_emb, S=S)
    assert np.array_equal(b1["part"].view(np.uint32), b2["part"].view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# forward + backward with a positional encoding: every first-layer layout, the ones column up to K's last
# ---------------------------------------------------------------------------------------------------------------------
def pe_x(rng, n, d, nfreq, fmt):
    """x on the grid 1/128 (|x| <= 2) whose sines all lie farther than SIN_TOL from a 16-bit midpoint (so the operand is
    r(sin)) and have |sin| >= 1/4 (so every operand is a multiple of 2^-13 and the dW0 sums fit 24 bits)."""
    xs = dyadic(rng, (60 * n, d), 256, 128)
    s = R.sin_values(xs, d, nfreq)
    sine = np.array([fr != 0 for _, fr in R.pe_columns(d, nfreq)], bool)
    ok = R.pe_exact(xs, d, nfreq, fmt) & (np.abs(s[:, sine]) >= 0.25).all(1)
    assert ok.sum() >= n
    return xs[ok][:n]


@pytest.mark.parametrize("route", ["fp32", "d16"])
@pytest.mark.parametrize("fmt", FMTS)
def test_pe_layouts_forward_and_backward(fmt, route):
    """The backward's producer builds its own [pe | 1] (write_a0_row, dib_sin_pe); dW0 / db0 are flushed from column w_in of
    the dW0p accumulator, at w_in = 14 and 15 the last columns of K.  W0 is 0 (the hidden activations come from b0 through
    the ones column, so the forward's sums stay on a coarse grid; the forward's operand is read out by
    test_pe_operand_exact_where_the_sine_is_far_from_a_midpoint) and the gradient operands are integers (beta = 0), so
    every dW0 sum over the fine-grained [pe | 1] operand fits 24 bits (asserted)."""
    rng = np.random.default_rng(12)
    n = 130
    for d, nfreq in LAYOUTS:
        enc = R.exact_params(rng, (d,), nfreq, -3.0, 1 / 32)
        enc[0]["W0"][:] = 0.0
        c = make_case(fmt, (d,), nfreq, "relu", n, x=[pe_x(rng, n, d, nfreq, fmt)], enc=enc)
        eps = dyadic(rng, (n, 1, R.E), 2, 1)
        S = loss_scale(n)
        d_emb = (2 * dyadic(rng, (n, R.E), 1, 1) / S).astype(np.float32)
        g = (d_emb * np.float32(S)).astype(np.float64)
        kw = dict(d_emb=d_emb) if route == "fp32" else dict(d_emb16=g)
        for grid in (1, 2):
            out = run(c, 7, grid, eps=eps, beta=0.0, S=S, inv_batch=1.0 / S, **kw)
            what = f"{fmt} pe layout d={d} nfreq={nfreq} grid={grid} {route}"
            check_pack(c, out)
            ref = check_forward(c, out, eps, what)
            check_backward(c, out, ref, eps, g, 0.0, what)


# ---------------------------------------------------------------------------------------------------------------------
# the bounded regime: lv != 0, the SFU activations, leaky ReLU with alpha = 0.2
# ---------------------------------------------------------------------------------------------------------------------
def within_silent(got, want, bound, what):
    """|got - want| <= bound everywhere; elements with a zero bound equal the reference by value.  Records the worst
    measured / bound of the inexact elements in WORST under the output's name."""
    err = np.abs(got - want)
    ok = err <= bound
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements outside the bound, first at {i}: got {got[i]!r}, want "
                             f"{want[i]!r} +- {bound[i]!r}")
    inexact = bound > 0
    if inexact.any():
        key = what.split(":")[0]
        WORST[key] = max(WORST.get(key, 0.0), float((err[inexact] / bound[inexact]).max()))


BOUNDED = [("tanh", "fp16", "fp32", 0.25), ("tanh", "bf16", "d16", 0.25), ("sigmoid", "fp16", "d16", 0.25),
           ("sigmoid", "bf16", "fp32", 0.25), ("elu", "fp16", "fp32", 0.25), ("elu", "bf16", "d16", 0.25),
           ("relu", "fp16", "d16", 0.25), ("relu", "bf16", "fp32", 0.25), ("linear", "fp16", "fp32", 0.25),
           ("leaky_relu", "bf16", "d16", 0.25), ("leaky_relu", "fp16", "fp32", 0.2), ("leaky_relu", "bf16", "d16", 0.2)]


@pytest.mark.parametrize("grid", [0, 2])
@pytest.mark.parametrize("act,fmt,route,alpha", BOUNDED)
def test_bounded_regime(act, fmt, route, alpha, grid):
    """lv != 0 (W2's logvar columns and b2's logvar half live, a non-dyadic logvar_offset): sv = __expf(lv / 2), the KL
    term sv^2 - lv - 1, the backward's expf(lv / 2) and dl's KL term; tanh / sigmoid / elu in frag_to_a and
    frag_dgrad_to_a; leaky ReLU with alpha = 0.2.  Every output within its bound (enc_fused_reference.bounded_*)."""
    rng = np.random.default_rng(21)
    fdims, n = (1, 3, 2), 300
    enc = R.bounded_params(rng, fdims, 1, -1.3)
    c = make_case(fmt, fdims, 1, act, n, seed=22, logvar_offset=-1.3, enc=enc, alpha=alpha)
    eps, d_emb, S = exact_inputs(c, 23)
    g = (d_emb * np.float32(S)).astype(np.float64)
    kw = dict(d_emb=d_emb) if route == "fp32" else dict(d_emb16=g)
    beta = 0.75
    out = run(c, 7, grid, eps=eps, beta=beta, S=S, inv_batch=1.0 / S, **kw)
    F, E = c.F, R.E
    ref = R.bounded_forward(c.img, c.x, c.x_off, c.fdims, 1, act, alpha, fmt, n, eps, out["g_fwd"])
    assert np.abs(np.concatenate([ch["lv"] for ch in ref["chains"]])).max() > 1.0, "the case needs a live logvar"
    tag = f"{act} a={alpha}"
    assert np.all(out["emb"][n:] == SENT32) and np.all(out["emb16"][n:] == SENT16) and np.all(out["user"][n:] == SENT32)
    within_silent(out["user"][:n].astype(np.float64), ref["user_emb"], ref["user_emb_bound"], f"{tag} user_emb: {fmt} grid {grid}")
    within_silent(out["emb"][:n, :F * E].astype(np.float64), ref["emb"], ref["emb_bound"], f"{tag} emb: {fmt} grid {grid}")
    within_silent(from16(out["emb16"][:n, :F * E], fmt), ref["emb16"], ref["emb16_bound"], f"{tag} emb16: {fmt} grid {grid}")
    kl, klb = np.zeros(out["kl"].shape), np.zeros(out["kl"].shape)
    kl[:, :ref["kl_part"].shape[1]], klb[:, :ref["kl_part"].shape[1]] = ref["kl_part"], ref["kl_part_bound"]
    within_silent(out["kl"].astype(np.float64), kl, klb, f"{tag} kl_part: {fmt} grid {grid}")
    parts = R.bounded_backward(c.img, ref["chains"], c.fdims, 1, act, alpha, fmt, n, eps, g, beta, 1.0 / S, S, out["g_bwd"])
    want, bound = R.bounded_partial_table(parts, c.lay, out["split_stride"], out["slots"] + 1, float(SENT32))
    within_silent(out["part"].astype(np.float64), want, bound, f"{tag} partials: {fmt} grid {grid} {route}")


# ---------------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_hook_rejects_bad_arguments():
    """Each host check refuses its argument before anything is launched (run() raises with the hook's message)."""
    c = make_case("fp16", (1, 2), 1, "relu", 200)
    eps, d_emb, S = exact_inputs(c)
    g = (d_emb * np.float32(S)).astype(np.float64)
    plus = lambda k: (lambda p: ctypes.c_void_p(p.value + k))
    cases = [(dict(grid=5), {}, "grid"), (dict(S=3.0), {}, "gscale"),
             ({}, dict(emb=plus(4)), "emb must be 8-byte aligned"), ({}, dict(ldemb=65), "emb must be"),
             ({}, dict(user_emb=plus(4)), "user_emb"), ({}, dict(emb16=plus(2)), "emb16 must be"),
             ({}, dict(eps=plus(4)), "eps must be"), ({}, dict(kl_stride=0), "kl_stride"),
             ({}, dict(part=plus(4)), "part 8-byte"), ({}, dict(split_stride=lambda v: v - 70), "inside params and split_stride"),
             ({}, dict(param_count=lambda v: v - 70), "parameter block b2_off"), ({}, dict(ldx=3), "x columns of feature 1"),
             ({}, dict(d_emb=plus(4)), "d_emb must be"), ({}, dict(ldd=63), "d_emb must be"),
             ({}, dict(phases=8), "phases"), ({}, dict(act=9), "unknown act")]
    for kw, over, msg in cases:
        with pytest.raises(AssertionError, match=msg):
            run(c, 7, eps=eps, d_emb=d_emb, S=kw.get("S", S), grid=kw.get("grid", 0), over=over)
    for over, msg in ((dict(d_emb16=plus(2)), "d_emb16 must be"), (dict(ldd16=68), "d_emb16 must be"),
                      (dict(ldd16=56), "d_emb16 must be")):
        with pytest.raises(AssertionError, match=msg):
            run(c, 7, eps=eps, d_emb16=g, S=S, over=over)
    with pytest.raises(AssertionError, match="exactly one of d_emb and d_emb16"):
        run(c, 7, eps=eps, d_emb=d_emb, d_emb16=g, S=S)
    c2 = make_case("fp16", (3,), 5, "relu", 10)
    c2.nfreq = 6
    with pytest.raises(AssertionError, match="fdim nfreq"):
        run(c2, 1)


def test_zz_report_worst_ratios():
    for k, v in sorted(WORST.items()):
        print(f"worst measured / bound  {k}: {v:.3g}")
