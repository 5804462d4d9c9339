"""GPU (H100): the set-transformer kernels element by element against the float64 reference with per-element bounds
(tests/set_attention_reference.py): the fixed-size and the key-tiled attention forward and backward, LayerNorm forward and
backward, mean pooling and zero_pad_rows, through the test hooks dib_debug_set_attention / dib_debug_layer_norm /
dib_debug_set_pool, which launch them as the training step does.  Every call also checks the memory contracts: NaN in every
input element a kernel must not read, a sentinel in every output element it must not write, and the launch count."""
import ctypes

import numpy as np
import pytest
import torch

from tests import set_attention_reference as R

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-3.0e33)
WORST = {}
ACT = {a: i for i, a in enumerate(R.ACTS)}


def _lib():
    from dib_b200 import _lib as L
    return L, L.load()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def within(what, got, ref, bound, tag):
    got, ref, bound = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.asarray(bound, np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{tag} {what}: {bad.sum()} of {bad.size} elements outside their bound; first at "
                           f"{np.argwhere(bad)[0].tolist()}: got {got[bad][0]!r} ref {ref[bad][0]!r} bound {bound[bad][0]!r}")
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    WORST[what] = max(WORST.get(what, 0.0), ratio)
    print(f"{tag} {what}: worst measured / bound {ratio:.3g}; exact elements {int((~pos).sum())}")


# ---- attention ----------------------------------------------------------------------------------------------------------
def _row_mask(sizes, S, L):
    l = np.full(S, L) if sizes is None else np.clip(np.asarray(sizes), 1, L)
    return (np.arange(L)[None, :] < l[:, None]).reshape(S * L)


def _rows_in(x, ld, real):
    """[S, H, L, dk] -> device [S * L, ld] rows: NaN in the columns past heads * dk and in the padding rows"""
    m = R.merge_heads(np.asarray(x, np.float32))
    buf = np.full((max(m.shape[0], 1), ld), np.nan, np.float32)      # sets = 0: a valid pointer all the same
    buf[:m.shape[0], :m.shape[1]] = m
    buf[:m.shape[0]][~real] = np.nan
    return _dev(buf)


def attention(variable, q, k, v, g=None, sizes=None, phases=3, o_in=None, lse_in=None, round_out=0, ld_extra=3, raw_sizes=None):
    """One hook call (or two with phases 1 then 2 fed o_in / lse_in): q, k, v, g [S, H, L, dk] fp32 -> dict of outputs in the
    head-split layout.  Checks the untouched columns / rows / slots and the launch count."""
    L_, lib = _lib()
    S, H, L, dk = q.shape
    ld = H * dk + ld_extra
    real = _row_mask(sizes, S, L) if variable else np.ones(S * L, bool)
    Q, K, V = (_rows_in(t, ld, real) for t in (q, k, v))
    bwd = bool(phases & 2)
    G = _rows_in(g, ld, real) if bwd else None
    n_h = S * H * L
    if o_in is not None:
        O_ = _rows_in(o_in, ld, real)
        lse = _dev(np.concatenate([np.where(real.reshape(S, 1, L), np.asarray(lse_in, np.float32), np.nan).reshape(-1),
                                   np.full(40, SENTINEL, np.float32)]))
    else:
        O_ = _dev(np.full((S * L + 1, ld), SENTINEL, np.float32))
        lse = _dev(np.full(n_h + 40, SENTINEL, np.float32))
    outs = {n: _dev(np.full((S * L + 1, ld), SENTINEL, np.float32)) for n in ("dq", "dk", "dv")} if bwd else {}
    dsum = _dev(np.full(n_h + 40, SENTINEL, np.float32)) if variable else None
    sz = None
    if variable:
        sz = _dev(np.asarray(sizes if raw_sizes is None else raw_sizes, np.int32).reshape(-1)[:max(S, 1)] if S else np.ones(1, np.int32))
    p = L_.ptr
    before = int(lib.dib_launch_count())
    L_.check(lib.dib_debug_set_attention(variable, phases, p(Q), p(K), p(V), p(G), ld, S, H, L, dk, p(sz), p(O_), p(lse),
                                         p(outs.get("dq")), p(outs.get("dk")), p(outs.get("dv")), p(dsum), round_out, _st()))
    want = 0 if S == 0 else (phases & 1) + ((2 if variable else 1) if bwd else 0)
    assert int(lib.dib_launch_count()) - before == want
    res = {}
    names = (["o"] if phases & 1 else []) + list(outs)
    bufs = dict(o=O_, **outs)
    for n in names:
        b = bufs[n].cpu().numpy()
        assert np.all(b[S * L:] == SENTINEL), f"{n}: a row past sets * L was written"
        assert np.all(b[:, H * dk:] == SENTINEL), f"{n}: a column past heads * dk was written"
        res[n] = R.split_heads(b[:S * L], S, L, H, dk)
    lv = lse.cpu().numpy()
    assert np.all(lv[n_h:] == SENTINEL), "lse: a slot past sets * heads * L was written"
    res["lse"] = lv[:n_h].reshape(S, H, L)
    if dsum is not None:
        dv_ = dsum.cpu().numpy()
        assert np.all(dv_[n_h:] == SENTINEL), "dsum: a slot past sets * heads * L was written"
        if bwd:
            res["dsum"] = dv_[:n_h].reshape(S, H, L)
        else:
            assert np.all(dv_ == SENTINEL)
    return res


def reference(q, k, v, g, sizes, o_in, lse_in):
    """R.attention_forward and R.attention_backward (from o_in / lse_in) over set chunks, concatenated"""
    S, H, L, dk = q.shape
    chunk = max(1, 2 ** 24 // (H * L * L * dk))
    f, b = {}, {}
    for s0 in range(0, max(S, 1), chunk):
        sl = slice(s0, s0 + chunk)
        sz = None if sizes is None else np.asarray(sizes)[sl]
        ff = R.attention_forward(q[sl], k[sl], v[sl], sz)
        bb = R.attention_backward(q[sl], k[sl], v[sl], g[sl], o_in[sl], lse_in[sl], sz) if g is not None else {}
        for dst, src in ((f, ff), (b, bb)):
            for key in src:
                if key.endswith("bound") or key in ("o", "lse", "dq", "dk", "dv", "dsum"):
                    dst.setdefault(key, []).append(src[key])
    return ({k_: np.concatenate(v_) for k_, v_ in f.items()}, {k_: np.concatenate(v_) for k_, v_ in b.items()})


def check_attention(variable, q, k, v, g, sizes, tag, from_float64=False):
    """forward and backward of one case within their bounds; the backward from the kernel's own o / lse, or (from_float64)
    from the float64 o / lse rounded to fp32.  Returns the kernel outputs."""
    if from_float64:
        f, _ = reference(q, k, v, None, sizes, None, None)
        o_in, lse_in = f["o"].astype(np.float32), f["lse"].astype(np.float32)
        out = attention(variable, q, k, v, g, sizes, phases=2, o_in=o_in, lse_in=lse_in)
    else:
        out = attention(variable, q, k, v, g, sizes, phases=3)
        o_in, lse_in = out["o"], out["lse"]
    f, b = reference(q, k, v, g, sizes, o_in, lse_in)
    kind = "varlen" if variable else "fixed"
    if not from_float64:
        within(f"{kind} o", out["o"], f["o"], f["o_bound"], tag)
        within(f"{kind} lse", out["lse"], f["lse"], f["lse_bound"], tag)
    for n in ("dq", "dk", "dv") + (("dsum",) if variable else ()):
        within(f"{kind} {n}", out[n], b[n], b[n + "_bound"], tag)
    return out


FIXED_L = (1, 2, 31, 32, 33, 50, 63, 64)
FIXED_HD = ((4, 1), (3, 12), (4, 17), (4, 33), (2, 64), (4, 127), (12, 128))


@pytest.mark.parametrize("heads,dk", FIXED_HD)
@pytest.mark.parametrize("L", FIXED_L)
def test_fixed_shapes(L, heads, dk):
    q, k, v, g = R.attention_case(3, heads, L, dk, seed=21)
    out = check_attention(0, q, k, v, g, None, f"fixed L={L} h={heads} dk={dk}")
    if L == 1:
        np.testing.assert_array_equal(out["o"], v)


@pytest.mark.parametrize("sets", [32, 1024])
def test_fixed_notebook_shape(sets):
    q, k, v, g = R.attention_case(sets, 12, 50, 128, seed=22)
    check_attention(0, q, k, v, g, None, f"fixed notebook sets={sets}")


VAR_LMAX = (1, 7, 63, 64, 65, 100, 128, 129, 256)
VAR_DK = (1, 12, 16, 17, 33, 100, 128)


def var_sizes(Lmax, seed=0):
    base = [s for s in (1, 63, 64, 65, 127, 128, 129) if s <= Lmax] + [Lmax]
    rng = np.random.default_rng([seed, Lmax])
    return np.array(base + list(rng.integers(1, Lmax + 1, size=2)), np.int32)


@pytest.mark.parametrize("dk", VAR_DK)
@pytest.mark.parametrize("Lmax", VAR_LMAX)
def test_varlen_shapes(Lmax, dk):
    sizes = var_sizes(Lmax)
    heads = 4 if dk % 4 else 1
    q, k, v, g = R.attention_case(len(sizes), heads, Lmax, dk, seed=23)
    out = check_attention(1, q, k, v, g, sizes, f"varlen Lmax={Lmax} dk={dk}")
    one = sizes == 1
    np.testing.assert_array_equal(out["o"][one, :, :1], v[one, :, :1])        # l = 1: O = V exactly


@pytest.mark.parametrize("variable", [0, 1])
@pytest.mark.parametrize("sets", [1, 7, 65535])
def test_set_counts(variable, sets):
    rng = np.random.default_rng(sets)
    q, k, v, g = R.attention_case(sets, 4, 2, 1, seed=24)
    sizes = rng.integers(1, 3, size=sets).astype(np.int32) if variable else None
    check_attention(variable, q, k, v, g, sizes, f"{'varlen' if variable else 'fixed'} sets={sets}")


@pytest.mark.parametrize("variable", [0, 1])
def test_zero_sets_launch_nothing(variable):
    q = np.zeros((0, 4, 8, 3), np.float32)
    out = attention(variable, q, q, q, q, np.zeros(0, np.int32) if variable else None)
    assert out["o"].size == 0 and out["lse"].size == 0


@pytest.mark.parametrize("dgrad", ["random", "dO=O", "dO_perp_O"])
@pytest.mark.parametrize("regime", R.REGIMES)
@pytest.mark.parametrize("variable", [0, 1])
def test_regimes(variable, regime, dgrad):
    L, heads, dk = (50, 4, 17) if not variable else (129, 1, 16)
    if regime == "dyadic":
        dk = 16
    sizes = None if not variable else np.array([129, 65, 1, 100, 64], np.int32)
    S = 3 if not variable else len(sizes)
    q, k, v, g = R.attention_case(S, heads, L, dk, regime, seed=25)
    if dgrad != "random":
        o64 = reference(q, k, v, None, sizes, None, None)[0]["o"]
        if dgrad == "dO=O":
            g = o64.astype(np.float32)
        else:
            gg = g.astype(np.float64)
            nn = np.maximum((o64 * o64).sum(-1, keepdims=True), 1e-30)
            g = (gg - (gg * o64).sum(-1, keepdims=True) / nn * o64).astype(np.float32)
    tag = f"{'varlen' if variable else 'fixed'} {regime} {dgrad}"
    if regime == "wide":
        s = R.attention_forward(q, k, v, sizes)["s"]
        s = np.where(np.isfinite(s), s, np.nan)
        assert np.nanmax(np.nanmax(s, -1) - np.nanmin(s, -1)) > 100
    if regime == "flat":
        assert np.all(q == 0)
    check_attention(variable, q, k, v, g, sizes, tag)
    check_attention(variable, q, k, v, g, sizes, tag + " (float64 o / lse)", from_float64=True)


@pytest.mark.parametrize("L", [8, 33, 50, 64])
def test_varlen_at_uniform_sizes_and_the_fixed_kernel_each_within_its_bound(L):
    q, k, v, g = R.attention_case(5, 4, L, 17, seed=26)
    check_attention(0, q, k, v, g, None, f"fixed L={L}")
    check_attention(1, q, k, v, g, np.full(5, L, np.int32), f"varlen uniform l={L}")


@pytest.mark.parametrize("variable", [0, 1])
def test_attention_identities(variable):
    """repeated calls are bit-identical; the backward alone from the forward's o / lse reproduces phases 3; round_out = rna of
    the round_out = 0 outputs given the same inputs (lse / dsum untouched; a rounded o changes D, so the backward's check
    feeds both the same o); permuted sets and heads permute the outputs."""
    S, H, L, dk = 6, 4, (50 if not variable else 129), 17
    sizes = None if not variable else np.array([129, 1, 64, 65, 100, 7], np.int32)
    q, k, v, g = R.attention_case(S, H, L, dk, seed=27)
    base = attention(variable, q, k, v, g, sizes)
    again = attention(variable, q, k, v, g, sizes)
    for n in base:
        np.testing.assert_array_equal(again[n], base[n], err_msg=n)
    fwd = attention(variable, q, k, v, None, sizes, phases=1, round_out=1)
    np.testing.assert_array_equal(fwd["o"], R.round_tf32(base["o"]))
    np.testing.assert_array_equal(fwd["lse"], base["lse"])
    b0 = attention(variable, q, k, v, g, sizes, phases=2, o_in=base["o"], lse_in=base["lse"])
    b1 = attention(variable, q, k, v, g, sizes, phases=2, o_in=base["o"], lse_in=base["lse"], round_out=1)
    for n in b0:
        if n == "lse":
            continue
        np.testing.assert_array_equal(b0[n], base[n], err_msg=f"backward alone {n}")
        want = b0[n] if n == "dsum" else R.round_tf32(b0[n])
        np.testing.assert_array_equal(b1[n], want, err_msg=f"round_out {n}")
    sp, hp = np.array([3, 0, 5, 1, 4, 2]), np.array([2, 0, 3, 1])
    perm = attention(variable, *(t[sp][:, hp] for t in (q, k, v, g)), None if sizes is None else sizes[sp])
    for n in base:
        np.testing.assert_array_equal(perm[n], base[n][sp][:, hp], err_msg=f"permuted {n}")


def test_varlen_set_does_not_depend_on_lmax():
    q, k, v, g = R.attention_case(2, 4, 256, 17, seed=28)
    sizes = np.array([70, 100], np.int32)
    big = attention(1, q, k, v, g, sizes)
    small = attention(1, *(t[:, :, :100] for t in (q, k, v, g)), sizes)
    for n in small:
        np.testing.assert_array_equal(big[n][:, :, :100], small[n], err_msg=n)
        assert np.all(big[n][:, :, 100:] == 0.0), n


def test_out_of_range_sizes_are_the_nearest_bound_in_every_kernel():
    """set sizes 0 and -5 act as 1, Lmax + 1 as Lmax: attention, masked pooling, the LayerNorm's pooled gradient and
    zero_pad_rows agree with the in-range sizes bit for bit."""
    L_, lib = _lib()
    Lmax, H, dk, E = 65, 4, 17, 36
    bad, good = np.array([0, -5, Lmax + 1, 3], np.int32), np.array([1, 1, Lmax, 3], np.int32)
    q, k, v, g = R.attention_case(4, H, Lmax, dk, seed=29)
    a = attention(1, q, k, v, g, good)
    b = attention(1, q, k, v, g, good, raw_sizes=bad)
    for n in a:
        np.testing.assert_array_equal(b[n], a[n], err_msg=n)
    rng = np.random.default_rng(30)
    x = rng.standard_normal((4 * Lmax, 40)).astype(np.float32)
    np.testing.assert_array_equal(pool(x, Lmax, E, bad), pool(x, Lmax, E, good))
    np.testing.assert_array_equal(zero_pad(x, Lmax, bad), zero_pad(x, Lmax, good))
    case = ln_case(4 * Lmax, E, 40, seed=31)
    dpool = rng.standard_normal((4, 40)).astype(np.float32)
    kw = dict(dy_pool=dpool, pool_rows=Lmax, nsplit=3, rps=100)
    lb, lg = layer_norm(case, phases=3, sizes=bad, **kw), layer_norm(case, phases=3, sizes=good, **kw)
    for n in lg:
        np.testing.assert_array_equal(lb[n], lg[n], err_msg=n)


def test_out_of_range_sizes_are_the_nearest_bound_in_a_model_step():
    """the same through a whole variable-size step, whose reparameterisation forward and backward also read the sizes:
    gradients, statistics (the KL slot included) and predictions at sizes 0, -5 and Lmax + 1 equal those at 1, 1 and Lmax
    bit for bit.  The host check that rejects such sizes is bypassed to reach the kernels."""
    from tests.test_gpu_set_transformer_variable_sizes import case as model_case, make_model, small
    cfg = small(65)
    bad, good = np.array([0, -5, 66, 3, 65], np.int32), np.array([1, 1, 65, 3, 65], np.int32)
    p, x, y, eps, _ = model_case(cfg, good, 32)
    m = make_model(cfg)
    m.set_flat_weights(p)
    m.beta.assign(0.1)
    m._device_sizes = lambda sizes, n: torch.from_numpy(np.asarray(sizes, np.int32)).cuda()
    out = []
    for sizes in (good, bad):
        g, st = m.compute_gradients((x, sizes), y, eps=eps)
        pred = m((x, sizes), eps=eps)
        out.append((g.cpu().numpy(), st.cpu().numpy(), pred.cpu().numpy() if isinstance(pred, torch.Tensor) else np.asarray(pred)))
    for a, b, name in zip(out[0], out[1], ("gradients", "statistics", "predictions")):
        assert np.isfinite(a).all()
        np.testing.assert_array_equal(b, a, err_msg=name)


def test_attention_hook_rejects_what_the_library_cannot_run():
    L_, lib = _lib()
    buf = torch.zeros(1 << 16, device="cuda")
    sz = torch.ones(8, dtype=torch.int32, device="cuda")
    p = L_.ptr

    def call(variable=0, phases=3, ld=16, sets=2, heads=4, L=8, dk=4, sizes=sz, dsum=buf, dout=buf, o=buf):
        return lib.dib_debug_set_attention(variable, phases, p(buf), p(buf), p(buf), p(dout), ld, sets, heads, L, dk, p(sizes),
                                           p(o), p(buf), p(buf), p(buf), p(buf), p(dsum), 0, _st())
    for badargs in (dict(variable=2), dict(phases=0), dict(phases=4), dict(L=0), dict(L=65), dict(variable=1, L=257),
                    dict(dk=0), dict(dk=129), dict(heads=0), dict(ld=15),
                    dict(heads=3, dk=3), dict(sets=-1), dict(sets=65536),
                    dict(variable=1, sizes=None), dict(variable=1, dsum=None), dict(dout=None), dict(o=None)):
        assert call(**badargs) != 0, badargs
        assert lib.dib_last_error().startswith(b"dib_debug_set_attention"), lib.dib_last_error()
    assert call() == 0 and call(variable=1, L=8) == 0 and call(variable=1, phases=1, dsum=None) == 0


# ---- LayerNorm --------------------------------------------------------------------------------------------------------
def ln_case(rows, E, ld, seed=0, regime="normal", eps=1e-3):
    rng = np.random.default_rng([seed, rows, E])
    a = rng.standard_normal((rows, E))
    b = np.tanh(rng.standard_normal((rows, E)))
    if regime == "constant":
        a = np.repeat(rng.standard_normal((rows, 1)), E, 1)
        b = np.zeros((rows, E))
    elif regime == "offset":
        a = a + 1e4
    f32 = lambda t: np.asarray(t, np.float32)
    return dict(a=f32(a), b=f32(b), gamma=f32(rng.standard_normal(E)), beta=f32(rng.standard_normal(E)),
                dys=[f32(rng.standard_normal((rows, E))) for _ in range(4)], eps=float(np.float32(eps)), ld=ld, E=E, rows=rows)


def _ld_rows(x, ld, rows_alloc=None):
    x = np.asarray(x, np.float32)
    buf = np.full((x.shape[0] if rows_alloc is None else rows_alloc, ld), np.nan, np.float32)
    buf[:x.shape[0], :x.shape[1]] = x
    return _dev(buf)


def layer_norm(c, phases=3, srcs=(0, 1, 2, 3), dy_pool=None, pool_rows=1, sizes=None, act=None, alpha=0.2, nsplit=1, rps=None,
               round_out=0, mean_in=None, rstd_in=None, split_pad=5):
    """One dib_debug_layer_norm call; -> dict y, mean, rstd, d_res, d_branch, dgamma, dbeta (numpy, live columns)"""
    L_, lib = _lib()
    rows, E, ld = c["rows"], c["E"], c["ld"]
    rps = rows if rps is None else rps
    A, B = _ld_rows(c["a"], ld), _ld_rows(c["b"], ld)
    G, Be = _dev(c["gamma"]), _dev(c["beta"])
    full = lambda *shape: _dev(np.full(shape, SENTINEL, np.float32))
    Y = full(rows + 1, ld) if phases & 1 else None
    if phases & 1:
        M, Rs = full(rows + 8), full(rows + 8)
    else:
        M = _dev(np.concatenate([np.asarray(mean_in, np.float32), np.full(8, SENTINEL, np.float32)]))
        Rs = _dev(np.concatenate([np.asarray(rstd_in, np.float32), np.full(8, SENTINEL, np.float32)]))
    bwd = bool(phases & 2)
    dys = [_ld_rows(c["dys"][i], ld) if (bwd and i in srcs) else None for i in range(4)]
    DP = _ld_rows(dy_pool, ld) if (bwd and dy_pool is not None) else None
    SZ = _dev(np.asarray(sizes, np.int32)) if (bwd and sizes is not None) else None
    DR = full(rows + 1, ld) if bwd else None
    DB = full(rows + 1, ld) if (bwd and act is not None) else None
    stride = 2 * E + 2 * split_pad + 3          # gamma at [split_pad, +E), beta at [E + 2 split_pad, +E), the rest untouched
    goff, boff = split_pad, E + 2 * split_pad
    PART = full(nsplit + 2, stride) if bwd else None
    p = L_.ptr
    before = int(lib.dib_launch_count())
    L_.check(lib.dib_debug_layer_norm(phases, p(A), p(B), ld, rows, E, p(G), p(Be), c["eps"], p(Y), p(M), p(Rs),
                                      p(dys[0]), p(dys[1]), p(dys[2]), p(dys[3]), p(DP), pool_rows, p(SZ), p(DR), p(DB),
                                      ACT[act] if act is not None else 0, alpha, p(PART), stride, goff, boff, nsplit, rps,
                                      round_out, _st()))
    want = (1 if (phases & 1 and rows > 0) else 0) + (1 if bwd else 0)
    assert int(lib.dib_launch_count()) - before == want
    out = {}
    zcols = min(ld, 128)
    for n, buf in (("y", Y), ("d_res", DR), ("d_branch", DB)):
        if buf is None:
            continue
        v = buf.cpu().numpy()
        assert np.all(v[rows:] == SENTINEL), f"{n}: a row past rows was written"
        assert np.all(v[:rows, E:zcols] == 0.0), f"{n}: columns [E, min(ld, 128)) not zeroed"
        assert np.all(v[:rows, zcols:] == SENTINEL), f"{n}: a column past 128 was written"
        out[n] = v[:rows, :E]
    if phases & 1:
        for n, buf in (("mean", M), ("rstd", Rs)):
            v = buf.cpu().numpy()
            assert np.all(v[rows:] == SENTINEL), f"{n}: a slot past rows was written"
            out[n] = v[:rows]
    if bwd:
        v = PART.cpu().numpy()
        assert np.all(v[nsplit:] == SENTINEL), "part: a row past nsplit was written"
        outside = np.ones(stride, bool)
        outside[goff:goff + E] = outside[boff:boff + E] = False
        assert np.all(v[:, outside] == SENTINEL), "part: a column outside the gamma / beta ranges was written"
        out["dgamma"], out["dbeta"] = v[:nsplit, goff:goff + E], v[:nsplit, boff:boff + E]
    return out


def check_layer_norm(c, tag, srcs=(0, 1, 2, 3), dy_pool=None, pool_rows=1, sizes=None, act=None, nsplit=1, rps=None):
    out = layer_norm(c, 3, srcs, dy_pool, pool_rows, sizes, act, nsplit=nsplit, rps=rps)
    f = R.layer_norm_forward(c["a"], c["b"], c["gamma"], c["beta"], c["eps"])
    within("ln y", out["y"], f["y"], f["y_bound"], tag)
    within("ln mean", out["mean"], f["mean"], f["mean_bound"], tag)
    within("ln rstd", out["rstd"], f["rstd"], f["rstd_bound"], tag)
    pooled = R.pooled_dy(dy_pool, c["rows"], pool_rows, sizes) if dy_pool is not None else None
    b = R.layer_norm_backward(c["a"], c["b"], c["gamma"], out["mean"], out["rstd"], dys=[c["dys"][i] for i in srcs],
                              pooled=pooled, branch_act=act, alpha=float(np.float32(0.2)), nsplit=nsplit, rows_per_split=rps)
    within("ln d_res", out["d_res"], b["d_res"], b["d_res_bound"], tag)
    if act is not None:
        within("ln d_branch", out["d_branch"], b["d_branch"], b["d_branch_bound"], tag)
    within("ln dgamma", out["dgamma"], b["dgamma"], b["dgamma_bound"], tag)
    within("ln dbeta", out["dbeta"], b["dbeta"], b["dbeta_bound"], tag)
    return out, b


LN_E = (4, 8, 32, 36, 64, 100, 128)
LN_ROWS = (1, 7, 8, 9, 4097)


@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("E", LN_E)
def test_layer_norm_shapes(E, rows):
    eps = (0.0, 1e-6, 1e-3)[(LN_E.index(E) + LN_ROWS.index(rows)) % 3]
    ld = min(128, E + 4) if E < 128 else 128
    c = ln_case(rows, E, ld, seed=40, eps=eps)
    dpool = np.random.default_rng(41).standard_normal((-(-rows // 8), E)).astype(np.float32)
    check_layer_norm(c, f"ln E={E} rows={rows} eps={eps}", dy_pool=dpool, pool_rows=8,
                     act="relu", nsplit=max(1, -(-rows // 256)), rps=256)


@pytest.mark.parametrize("eps", [1e-6, 1e-3])
@pytest.mark.parametrize("regime", ["constant", "offset"])
@pytest.mark.parametrize("E", [36, 128])
def test_layer_norm_regimes(E, regime, eps):
    c = ln_case(33, E, E if E == 128 else 40, seed=42, regime=regime, eps=eps)
    out, _ = check_layer_norm(c, f"ln {regime} E={E} eps={eps}", act="tanh")
    if regime == "constant":
        assert np.all(np.abs(out["rstd"] - 1 / np.sqrt(eps)) <= 1e-3 / np.sqrt(eps))


SUBSETS = [tuple(i for i in range(4) if m >> i & 1) for m in range(16)]


@pytest.mark.parametrize("pool_kind", ["none", "fixed", "varlen"])
@pytest.mark.parametrize("srcs", SUBSETS)
def test_layer_norm_backward_sources(srcs, pool_kind):
    Lmax, S, E = 7, 3, 36
    c = ln_case(S * Lmax, E, 40, seed=43)
    dpool = None if pool_kind == "none" else np.random.default_rng(44).standard_normal((S, E)).astype(np.float32)
    sizes = np.array([1, 7, 4], np.int32) if pool_kind == "varlen" else None
    act = ([None] + list(R.ACTS))[SUBSETS.index(srcs) % 7]
    check_layer_norm(c, f"ln srcs={srcs} pool={pool_kind} act={act}", srcs, dpool, Lmax, sizes, act)


@pytest.mark.parametrize("act", [None] + list(R.ACTS))
def test_layer_norm_branch_activations(act):
    c = ln_case(21, 32, 32, seed=45)
    rng = np.random.default_rng(46)
    h = rng.standard_normal((21, 32))
    c["b"] = {"relu": np.maximum(h, 0), "tanh": np.tanh(h), "leaky_relu": np.where(h > 0, h, 0.2 * h),
              "sigmoid": 1 / (1 + np.exp(-h)), "elu": np.where(h > 0, h, np.expm1(h))}.get(act, h).astype(np.float32)
    c["b"][0, :4] = 0.0                            # h = 0: the derivative's side of the kink
    check_layer_norm(c, f"ln act={act}", act=act)


@pytest.mark.parametrize("rows,nsplit,rps", [(9, 1, 9), (4097, 1, 4097), (9, 3, 4), (4097, 5, 1000), (9, 5, 4), (1, 3, 1)])
def test_layer_norm_splits(rows, nsplit, rps):
    c = ln_case(rows, 36, 40, seed=47)
    out, _ = check_layer_norm(c, f"ln rows={rows} nsplit={nsplit} rps={rps}", nsplit=nsplit, rps=rps)
    empty = np.arange(nsplit) * rps >= rows
    assert np.all(out["dgamma"][empty] == 0.0) and np.all(out["dbeta"][empty] == 0.0)


def test_layer_norm_backward_alone_and_identities():
    """the backward alone from float64 mean / rstd rounded to fp32; round_out = rna of round_out = 0 (mean, rstd and the
    partials untouched); repeated calls bit-identical"""
    c = ln_case(50, 100, 104, seed=48)
    f = R.layer_norm_forward(c["a"], c["b"], c["gamma"], c["beta"], c["eps"])
    m32, r32 = f["mean"].astype(np.float32), f["rstd"].astype(np.float32)
    out = layer_norm(c, phases=2, mean_in=m32, rstd_in=r32, act="elu", nsplit=2, rps=25)
    b = R.layer_norm_backward(c["a"], c["b"], c["gamma"], m32, r32, dys=c["dys"], branch_act="elu", nsplit=2, rows_per_split=25)
    for n in ("d_res", "d_branch", "dgamma", "dbeta"):
        within(f"ln {n} (phase 2)", out[n], b[n], b[n + "_bound"], "ln backward alone")
    base = layer_norm(c, act="sigmoid", nsplit=2, rps=25)
    again = layer_norm(c, act="sigmoid", nsplit=2, rps=25)
    rounded = layer_norm(c, act="sigmoid", nsplit=2, rps=25, round_out=1)
    for n in base:
        np.testing.assert_array_equal(again[n], base[n], err_msg=n)
        want = R.round_tf32(base[n]) if n in ("y", "d_res", "d_branch") else base[n]
        np.testing.assert_array_equal(rounded[n], want, err_msg=f"round_out {n}")


def test_layer_norm_hook_rejects_what_the_library_cannot_run():
    L_, lib = _lib()
    buf = torch.zeros(1 << 14, device="cuda")
    p = L_.ptr

    def call(phases=3, ld=8, rows=4, E=8, eps=1e-3, pool=None, pool_rows=1, sizes=None, nsplit=1, rps=4, stride=16, goff=0,
             boff=8, act=0, branch=None, y=buf):
        return lib.dib_debug_layer_norm(phases, p(buf), p(buf), ld, rows, E, p(buf), p(buf), eps, p(y), p(buf), p(buf),
                                        None, None, None, None, p(pool), pool_rows, p(sizes), p(buf), p(branch), act, 0.2,
                                        p(buf), stride, goff, boff, nsplit, rps, 0, _st())
    for badargs in (dict(phases=0), dict(phases=4), dict(E=0), dict(E=129, ld=129), dict(E=6), dict(ld=7), dict(rows=-1),
                    dict(eps=-1.0), dict(eps=float("inf")), dict(nsplit=0), dict(rps=0), dict(nsplit=1, rps=3),
                    dict(goff=9), dict(boff=9), dict(goff=-1), dict(pool=buf, pool_rows=0), dict(sizes=buf),
                    dict(branch=buf, act=6), dict(y=None)):
        assert call(**badargs) != 0, badargs
        assert lib.dib_last_error().startswith(b"dib_debug_layer_norm"), lib.dib_last_error()
    assert call() == 0 and call(phases=2, y=None) == 0


# ---- pooling and zero_pad_rows ------------------------------------------------------------------------------------------
def pool(x, L, E, sizes=None, ldo=None, round_out=0):
    L_, lib = _lib()
    S = x.shape[0] // L
    ldo = E + 4 if ldo is None else ldo
    X = _dev(np.where(_row_mask(sizes, S, L)[:, None], x, np.nan).astype(np.float32))
    X[:, E:] = float("nan")
    out = _dev(np.full((S + 1, ldo), SENTINEL, np.float32))
    sz = _dev(np.asarray(sizes, np.int32)) if sizes is not None else None
    before = int(lib.dib_launch_count())
    L_.check(lib.dib_debug_set_pool(0, L_.ptr(X), x.shape[1], E, L, S, L_.ptr(sz), L_.ptr(out), ldo, round_out, _st()))
    assert int(lib.dib_launch_count()) - before == (1 if S else 0)
    v = out.cpu().numpy()
    assert np.all(v[S:] == SENTINEL) and np.all(v[:S, E:] == 0.0)
    return v[:S, :E]


def zero_pad(x, L, sizes):
    L_, lib = _lib()
    X = _dev(x)
    L_.check(lib.dib_debug_set_pool(1, L_.ptr(X), x.shape[1], 0, L, x.shape[0] // L, L_.ptr(_dev(np.asarray(sizes, np.int32))),
                                    None, 0, 0, _st()))
    return X.cpu().numpy()


@pytest.mark.parametrize("dyadic", [True, False])
@pytest.mark.parametrize("L,sizes", [(1, None), (8, None), (50, None), (64, None), (100, [1, 64, 37, 100, 0, 101]),
                                     (256, [256, 128, 129, 1, 255])])
def test_pooling(L, sizes, dyadic):
    rng = np.random.default_rng([50, L])
    S = 5 if sizes is None else len(sizes)
    x = rng.integers(-8, 9, size=(S * L, 40)) / 8.0 if dyadic else rng.standard_normal((S * L, 40))
    x = x.astype(np.float32)
    got = pool(x, L, 36, sizes)
    ref, bnd = R.pool(x[:, :36], L, sizes)
    within("pool", got, ref, bnd, f"pool L={L} sizes={sizes} dyadic={dyadic}")
    l = np.full(S, L) if sizes is None else np.clip(sizes, 1, L)
    if dyadic:
        exact = (l & (l - 1)) == 0
        np.testing.assert_array_equal(got[exact], ref[exact])
    np.testing.assert_array_equal(pool(x, L, 36, sizes, round_out=1), R.round_tf32(got))


def test_zero_pad_rows():
    rng = np.random.default_rng(51)
    Lmax, sizes = 100, np.array([1, 64, 100, 37], np.int32)
    x = rng.standard_normal((4 * Lmax, 12)).astype(np.float32)
    got = zero_pad(x, Lmax, sizes)
    real = _row_mask(sizes, 4, Lmax)
    np.testing.assert_array_equal(got[real], x[real])
    assert np.all(got[~real] == 0.0)


def test_pool_hook_rejects_what_the_library_cannot_run():
    L_, lib = _lib()
    buf = torch.zeros(1 << 14, device="cuda")
    sz = torch.ones(8, dtype=torch.int32, device="cuda")
    p = L_.ptr

    def call(zp=0, ld=8, E=8, L=4, sets=2, sizes=None, out=buf, ldo=8):
        return lib.dib_debug_set_pool(zp, p(buf), ld, E, L, sets, p(sizes), p(out), ldo, 0, _st())
    for badargs in (dict(zp=2), dict(zp=1), dict(L=0), dict(L=65), dict(L=257, sizes=sz), dict(sets=-1), dict(sets=65536),
                    dict(E=0), dict(E=129, ld=129, ldo=129), dict(E=6), dict(ld=7), dict(ldo=7), dict(out=None)):
        assert call(**badargs) != 0, badargs
        assert lib.dib_last_error().startswith(b"dib_debug_set_pool"), lib.dib_last_error()
    assert call() == 0 and call(L=200, sizes=sz) == 0 and call(zp=1, sizes=sz, out=None) == 0


def test_zz_print_worst_ratios():
    print("worst measured / bound over the file:", {k: round(v, 4) for k, v in sorted(WORST.items())})
