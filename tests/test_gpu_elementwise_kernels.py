"""GPU (H100): the elementwise kernels of the training step element by element against the float64 reference with per-element
bounds (tests/elementwise_reference.py): the compiled loss, the reparameterisation forward and backward with the KL partials,
the positional encoding, dropout and the fixed-order reductions, through the test hooks dib_debug_loss / dib_debug_reparam /
dib_debug_pe / dib_debug_dropout / dib_debug_reduce, which launch them as the training step does.  Every call also checks the
memory contracts: NaN in every input element a kernel must not read, a sentinel in every output element it must not write,
and the launch count."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import philox
from tests import elementwise_reference as R

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
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{tag} {what}: NaN where the reference has none, or the reverse"
    got, ref, bound = got[~nan], ref[~nan], bound[~nan]
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{tag} {what}: {bad.sum()} of {bad.size} elements outside their bound; first at "
                           f"{np.argwhere(bad)[0].tolist()}: got {got[bad][0]!r} ref {ref[bad][0]!r} bound {bound[bad][0]!r}")
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    WORST[what] = max(WORST.get(what, 0.0), ratio)
    print(f"{tag} {what}: worst measured / bound {ratio:.3g}; exact elements {int((~pos).sum())}")


def _launches(lib):
    return int(lib.dib_launch_count())


# ---- compiled loss ------------------------------------------------------------------------------------------------------
def run_loss(kind, act, z, y, inv_batch, w=None, alpha=0.2, round_out=0, ld_extra=3):
    """one dib_debug_loss call: z [n, C] fp32 -> dict of d_pred [n, C], user_pred, loss_part, acc_part; checks the memory
    contract (NaN in pred's pad columns, sentinels past every output) and the launch count"""
    L_, lib = _lib()
    n, C = z.shape
    ldp = C + ld_extra
    pred = np.full((n + 1, ldp), np.nan, np.float32)
    pred[:n, :C] = z
    dp = _dev(np.full((n + 1, ldp), SENTINEL, np.float32))
    up = _dev(np.full(n * C + 7, SENTINEL, np.float32))
    nblk = -(-n // 256)
    lp, ap = _dev(np.full(nblk + 3, SENTINEL, np.float32)), _dev(np.full(nblk + 3, SENTINEL, np.float32))
    yd = _dev(np.asarray(y, np.float32).reshape(-1))
    wd = _dev(np.asarray(w, np.float32)) if w is not None else None
    P = _dev(pred)
    before = _launches(lib)
    L_.check(lib.dib_debug_loss(R.LOSSES[kind], ACT[act], alpha, L_.ptr(P), ldp, L_.ptr(yd), C, n, inv_batch, L_.ptr(wd),
                                L_.ptr(dp), L_.ptr(up), L_.ptr(lp), L_.ptr(ap), round_out, _st()))
    assert _launches(lib) - before == (1 if n else 0)
    d = dp.cpu().numpy()
    assert np.all(d[n:] == SENTINEL), "d_pred: a row past n was written"
    assert np.all(d[:n, C:] == 0), "d_pred: the pad columns are not zeroed"
    u = up.cpu().numpy()
    assert np.all(u[n * C:] == SENTINEL)
    np.testing.assert_array_equal(u[:n * C].reshape(n, C), z)
    l, a = lp.cpu().numpy(), ap.cpu().numpy()
    assert np.all(l[nblk:] == SENTINEL) and np.all(a[nblk:] == SENTINEL)
    return dict(dz=d[:n, :C], loss_part=l[:nblk], acc_part=a[:nblk])


def check_loss(kind, act, z, y, inv_batch, tag, w=None, alpha=0.2):
    z = np.asarray(z, np.float32)
    out = run_loss(kind, act, z, y, inv_batch, w, alpha)
    ref = R.loss(kind, act, alpha, z, y, np.float32(inv_batch), w)
    within(f"{kind} dz", out["dz"], ref["dz"], ref["dz_bound"], tag)
    within(f"{kind} loss_part", out["loss_part"], ref["loss_part"], ref["loss_part_bound"], tag)
    within(f"{kind} acc_part", out["acc_part"], ref["acc_part"], ref["acc_part_bound"], tag)
    return out, ref


SPARSE_C = (1, 2, 3, 16, 17)


@pytest.mark.parametrize("C", SPARSE_C)
@pytest.mark.parametrize("weighted", [False, True])
def test_sparse_ce_labels_ties_and_edges(C, weighted):
    """labels 0, C - 1, -0.5, 2.7, -1, C and NaN; argmax ties; weights 0 and 1e6; n on either side of a 256-row block"""
    rng = np.random.default_rng(C)
    for n in (1, 255, 256, 257, 700):
        z = rng.standard_normal((n, C)).astype(np.float32) * 3
        z[::5] = np.round(z[::5])                                       # ties in the argmax
        z[::7, :] = 1.0                                                 # every output tied
        labels = np.array([0, C - 1, -0.5, 2.7, -1, C, np.nan], np.float32)
        y0 = rng.integers(0, C, n).astype(np.float32)
        edge = labels[:4][labels[:4] < C]                               # the edge labels valid for this C, in block 0
        y0[:min(n, edge.size)] = edge[:min(n, edge.size)]
        w = None
        if weighted:
            w = rng.uniform(0, 3, n).astype(np.float32)
            w[::3] = 0.0
            w[1::11] = 1e6
        check_loss("sparse_ce_logits", "linear", z, y0, 1.0 / n, f"C={C} n={n} w={weighted}", w)
        y = y0.copy()                                                   # the labels at the start of the last block only
        last = (n - 1) // 256 * 256
        k = min(7, n - last)
        y[last:last + k] = labels[[4, 5, 6, 0, 1, 2, 3]][:k]            # the invalid ones first
        out, ref = check_loss("sparse_ce_logits", "linear", z, y, 1.0 / n, f"C={C} n={n} w={weighted} invalid", w)
        bad = R.sparse_label(y, C) < 0
        assert np.isnan(out["dz"][bad]).all() and not np.isnan(out["dz"][~bad]).any()
        if n > 256:
            assert np.isfinite(out["loss_part"][:-1]).all() and np.isnan(out["loss_part"][-1])


@pytest.mark.parametrize("kind", ["bce_logits", "mse", "bce_probs"])
@pytest.mark.parametrize("C", [1, 3, 16, 17])
@pytest.mark.parametrize("act", R.ACTS)
def test_per_output_losses_at_kinks_and_saturation(kind, C, act):
    rng = np.random.default_rng(C * 7 + ACT[act])
    n = 513
    if kind == "bce_probs":
        z = rng.random((n, C)).astype(np.float32)
        z.flat[:6] = [0.0, R.KERAS_EPS, R.ONE_M_EPS, 1.0, 0.5, 1e-8]
    else:
        z = (rng.standard_normal((n, C)) * (30 if kind == "bce_logits" else 2)).astype(np.float32)
        z.flat[:8] = [80.0, -80.0, 0.0, -0.0, 1e-30, 0.5, 88.0, -88.0]
    if act in ("relu",):
        z = np.maximum(z, 0)
    elif act == "tanh":
        z = np.clip(z, -1, 1)
    elif act == "sigmoid":
        z = np.clip(np.abs(z), 0, 1)
    elif act == "elu":
        z = np.maximum(z, -1)
    y = (rng.random((n, C)) > 0.5).astype(np.float32) if kind != "mse" else rng.standard_normal((n, C)).astype(np.float32)
    w = rng.uniform(0, 2, n).astype(np.float32)
    w[:2] = [0.0, 1e6]
    check_loss(kind, act, z, y, 1.0 / n, f"{kind} C={C} {act}")
    check_loss(kind, act, z, y, 1.0 / n, f"{kind} C={C} {act} weighted", w)


def test_external_loss_applies_only_the_activation_derivative():
    rng = np.random.default_rng(3)
    z = np.tanh(rng.standard_normal((300, 5))).astype(np.float32)
    g = rng.standard_normal((300, 5)).astype(np.float32)
    out, _ = check_loss("external", "tanh", z, g, 1.0 / 300, "external")
    assert not out["loss_part"].any() and not out["acc_part"].any()


# ---- reparameterisation -----------------------------------------------------------------------------------------------
def run_reparam(mu, lv, eps=None, seed=0, step=0, step_dev=None, sample_offset=0, sizes=None, set_len=1, du=None, beta=0.5,
                inv_batch=1.0, round_out=0):
    """mu, lv [F, n, E] -> the hook's forward (and backward when du is given) outputs; checks the contracts"""
    L_, lib = _lib()
    F, n, E = mu.shape
    ldo, ldemb = 2 * E + 3, F * E + 2
    fs = n * ldo + 5
    enc = np.full(F * fs, np.nan, np.float32)
    for f in range(F):
        blk = np.full((n, ldo), np.nan, np.float32)
        blk[:, :E], blk[:, E:2 * E] = mu[f], lv[f]
        enc[f * fs:f * fs + n * ldo] = blk.reshape(-1)
    real = np.ones(n, bool)
    if sizes is not None:
        real = (np.arange(n) % set_len) < np.clip(np.repeat(sizes, set_len), 1, set_len)
        for f in range(F):       # the padding particles are never read
            v = enc[f * fs:f * fs + n * ldo].reshape(n, ldo)
            v[~real] = np.nan
    nblk = -(-n // 256)
    kls = nblk + 2
    emb = _dev(np.full((n + 1, ldemb), SENTINEL, np.float32))
    uemb = _dev(np.full(n * F * E + 5, SENTINEL, np.float32))
    klp = _dev(np.full(F * kls, SENTINEL, np.float32))
    Enc = _dev(enc)
    ed = None
    if eps is not None:
        ed = _dev(np.ascontiguousarray(np.transpose(eps, (1, 0, 2))).astype(np.float32))     # [n, F, E]
    sd = _dev(np.asarray(sizes, np.int32)) if sizes is not None else None
    sdv = _dev(np.asarray([step_dev], np.int32)) if step_dev is not None else None
    bwd = du is not None
    dud = dout = bd = None
    if bwd:
        d = np.full((n, ldemb), np.nan, np.float32)
        for f in range(F):
            d[:, f * E:(f + 1) * E] = du[f]
        dud = _dev(d)
        dout = _dev(np.full(F * fs, SENTINEL, np.float32))
        bd = _dev(np.asarray([beta], np.float32))
    p = L_.ptr
    before = _launches(lib)
    L_.check(lib.dib_debug_reparam(3 if bwd else 1, p(Enc), fs, ldo, F, E, n, p(ed), seed, step, p(sdv), sample_offset, p(sd),
                                   set_len, p(emb), ldemb, p(uemb), p(klp), kls, p(dud), p(bd), inv_batch, p(dout), round_out,
                                   _st()))
    assert _launches(lib) - before == ((2 if bwd else 1) if n else 0)
    e = emb.cpu().numpy()
    assert np.all(e[n:] == SENTINEL) and np.all(e[:n, F * E:] == 0)
    ue = uemb.cpu().numpy()
    assert np.all(ue[n * F * E:] == SENTINEL)
    k = klp.cpu().numpy().reshape(F, kls)
    assert np.all(k[:, nblk:] == SENTINEL)
    res = dict(emb=np.stack([e[:n, f * E:(f + 1) * E] for f in range(F)]),
               user_emb=np.stack([ue[:n * F * E].reshape(n, F, E)[:, f] for f in range(F)]), kl_part=k[:, :nblk], real=real)
    if bwd:
        o = dout.cpu().numpy()
        dm, dl = [], []
        for f in range(F):
            blk = o[f * fs:f * fs + n * ldo].reshape(n, ldo)
            assert np.all(blk[:, 2 * E:] == 0), "d_out: the pad columns are not zeroed"
            assert np.all(o[f * fs + n * ldo:(f + 1) * fs] == SENTINEL)
            dm.append(blk[:, :E]); dl.append(blk[:, E:2 * E])
        res.update(dmu=np.stack(dm), dlv=np.stack(dl))
    return res


def check_reparam(mu, lv, tag, eps=None, philox_key=None, sizes=None, set_len=1, du=None, beta=0.5, round_out=0):
    F, n, E = mu.shape
    if eps is not None:
        z, ztol, kw = eps, 0.0, {}
    else:
        seed, step, step_dev, off = philox_key
        z = np.transpose(philox.normal_noise(seed, step + (step_dev or 0), off + np.arange(n, dtype=np.uint64), F, E,
                                             dtype=np.float64), (1, 0, 2))
        ztol, kw = R.Z_TOL, dict(seed=seed, step=step, step_dev=step_dev, sample_offset=off)
    inv_batch = np.float32(1.0 / max(n, 1))
    out = run_reparam(mu, lv, eps, sizes=sizes, set_len=set_len, du=du, beta=beta, inv_batch=inv_batch, round_out=round_out, **kw)
    real = out["real"] if sizes is not None else None
    f = R.reparam_forward(mu, lv, z, ztol, real)
    within("reparam user_emb", out["user_emb"], f["u"], f["u_bound"], tag)
    eb = f["u_bound"] + (R.TF32_HALF_ULP * (np.abs(f["u"]) + f["u_bound"]) if round_out else 0)
    within("reparam emb", out["emb"], f["u"], eb, tag)
    within("reparam kl_part", out["kl_part"], f["kl_part"], f["kl_part_bound"], tag)
    if real is not None:
        assert np.all(out["user_emb"][:, ~real] == 0) and np.all(out["emb"][:, ~real] == 0)
    if du is not None:
        b = R.reparam_backward(mu, lv, z, du, beta, inv_batch, ztol, real)
        rb = (lambda r, bd: bd + (R.TF32_HALF_ULP * (np.abs(r) + bd) if round_out else 0))
        within("reparam dmu", out["dmu"], b["dmu"], rb(b["dmu"], b["dmu_bound"]), tag)
        within("reparam dlv", out["dlv"], b["dlv"], rb(b["dlv"], b["dlv_bound"]), tag)
    return out


@pytest.mark.parametrize("E", [1, 3, 4, 5, 32])
@pytest.mark.parametrize("F", [1, 3])
def test_reparam_shapes_with_eps_and_philox(E, F):
    rng = np.random.default_rng(E * 10 + F)
    for n in (1, 255, 256, 257, 4097):
        mu = rng.standard_normal((F, n, E)).astype(np.float32)
        lv = rng.standard_normal((F, n, E)).astype(np.float32) * 2
        lv.flat[:4] = [20.0, -20.0, 1e-4, -1e-4][:lv.size] if lv.size >= 4 else lv.flat[:4]
        du = rng.standard_normal((F, n, E)).astype(np.float32)
        eps = rng.standard_normal((F, n, E)).astype(np.float32)
        check_reparam(mu, lv, f"E={E} F={F} n={n} eps", eps=eps, du=du)
        check_reparam(mu, lv, f"E={E} F={F} n={n} philox", philox_key=(7, 3, 2, 2 ** 32 + 5), du=du, round_out=n == 257)


def test_philox_noise_against_normal_noise():
    """mu = lv = 0 makes u = fmaf(1, z, 0) = z: the kernel's Philox normals against oracle/philox.normal_noise, within
    R.Z_TOL (1 + |z|) without the factor C (the reference's u and d lv bounds take this tolerance as a first-order term)"""
    F, n, E = 3, 4097, 5
    zero = np.zeros((F, n, E), np.float32)
    out = run_reparam(zero, zero, seed=7, step=3, step_dev=2, sample_offset=2 ** 32 + 5)
    z = np.transpose(philox.normal_noise(7, 5, 2 ** 32 + 5 + np.arange(n, dtype=np.uint64), F, E, dtype=np.float64), (1, 0, 2))
    within("philox noise", out["user_emb"], z, R.Z_TOL * (1.0 + np.abs(z)), "philox")


@pytest.mark.parametrize("s", [1e-4, 1e-3])
def test_kl_where_features_switch_off(s):
    """mu, lv ~ N(0, s^2): the regime high beta drives unused features into; the KL partials keep their relative accuracy"""
    rng = np.random.default_rng(11)
    mu = (rng.standard_normal((2, 4096, 4)) * s).astype(np.float32)
    lv = (rng.standard_normal((2, 4096, 4)) * s).astype(np.float32)
    du = rng.standard_normal(mu.shape).astype(np.float32)
    out = check_reparam(mu, lv, f"small s={s}", eps=np.zeros_like(mu), du=du, beta=1000.0)
    ref = R.reparam_forward(mu, lv, np.zeros_like(mu))
    assert np.abs(out["kl_part"] - ref["kl_part"]).max() <= 1e-5 * np.abs(ref["kl_part"]).max()


def test_reparam_padded_sets():
    rng = np.random.default_rng(12)
    L, S, E, F = 8, 70, 4, 1
    n = L * S
    sizes = rng.integers(1, L + 1, S)
    sizes[:3] = [0, L + 5, 1]                                          # clamped into [1, L]
    mu = rng.standard_normal((F, n, E)).astype(np.float32)
    lv = rng.standard_normal((F, n, E)).astype(np.float32)
    du = rng.standard_normal((F, n, E)).astype(np.float32)
    out = check_reparam(mu, lv, "padded eps", eps=rng.standard_normal((F, n, E)).astype(np.float32), sizes=sizes, set_len=L, du=du)
    assert np.all(out["dmu"][:, ~out["real"]] == 0) and np.all(out["dlv"][:, ~out["real"]] == 0)
    check_reparam(mu, lv, "padded philox", philox_key=(3, 1, 4, 2 ** 33), sizes=sizes, set_len=L, du=du)


# ---- positional encoding ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gather", [False, True])
def test_pe_columns_frequencies_and_row_clamp(gather):
    L_, lib = _lib()
    rng = np.random.default_rng(13)
    n, d, ldx = 1000, 3, 6
    x = np.full((n, ldx), np.nan, np.float32)
    x[:, 1:1 + d] = rng.uniform(-1e3, 1e3, (n, d)).astype(np.float32)
    x[:5, 1:1 + d] = [[0.0, -0.0, 1e-30], [1e3, -1e3, 3.14159], [1.0, 2.0, 0.5], [1e-3, 5e2, -7.0], [40.0, 80.0, 160.0]]
    freqs = [0, 2, 4, 8, 16]
    col_src = np.array([-1] + [1 + k for f in freqs for k in range(d)] + [-1, -1], np.int32)     # x_col_shift = 0: columns 1..3
    col_freq = np.array([0] + [f for f in freqs for _ in range(d)] + [0, 0], np.int32)
    ncol = len(col_src)
    col_begin, col_end, shift = 1, ncol, 1
    ldpe = ncol + 2
    row_index = col_feat = None
    n_src = n
    if gather:
        col_feat = np.array([0] + [k for _ in freqs for k in range(d)] + [0, 0], np.int32)
        row_index = rng.integers(-5, n + 5, (d, n)).astype(np.int32)         # outside [0, n_src) clamps
    out = _dev(np.full((n + 1, ldpe), SENTINEL, np.float32))
    p = L_.ptr
    ri, cf = (_dev(row_index), _dev(col_feat)) if gather else (None, None)
    X, CS, CF = _dev(x), _dev(col_src), _dev(col_freq)
    before = _launches(lib)
    L_.check(lib.dib_debug_pe(p(X), ldx, 0, p(CS), p(CF), col_begin, col_end, p(out), ldpe, shift, n, p(ri), p(cf), n_src, 0,
                              _st()))
    assert _launches(lib) - before == 1
    o = out.cpu().numpy()
    assert np.all(o[n:] == SENTINEL) and np.all(o[:, col_end - shift:] == SENTINEL)
    ref, b = R.pe(x, col_src, col_freq, col_begin, col_end, 0, row_index, col_feat, n_src, n)
    within("pe", o[:n, :col_end - shift], ref, b, f"pe gather={gather}")
    assert np.all(o[:n, col_end - shift - 2:col_end - shift] == 0)            # col_src = -1 columns


# ---- dropout ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", [0.0, 2.0 ** -24, 0.5, 0.3])
@pytest.mark.parametrize("width", [1, 6, 13, 64])
def test_dropout_masks_are_bit_exact(rate, width):
    L_, lib = _lib()
    rng = np.random.default_rng(width)
    F, n, ld = 3, 300, width + 3
    fs = n * ld + 4
    seed, step, step_dev, off, layer = 2 ** 40 + 9, 5, 3, 2 ** 32 + 1, 2
    src = np.full(F * fs, np.nan, np.float32)
    vals = rng.standard_normal((F, n, width)).astype(np.float32)
    for f in range(F):
        v = src[f * fs:f * fs + n * ld].reshape(n, ld)
        v[:, :width] = vals[f]
    sdv = _dev(np.asarray([step_dev], np.int32))
    for feature in (-1, 1):
        for backward in (0, 1):
            dst0 = np.full(F * fs, SENTINEL, np.float32)
            if backward:
                dst0[:] = src
            dst, S = _dev(dst0), _dev(src)
            before = _launches(lib)
            L_.check(lib.dib_debug_dropout(None if backward else L_.ptr(S), L_.ptr(dst), fs, ld, width, F, n, rate,
                                           seed, step, L_.ptr(sdv), off, layer, feature, backward, 0, _st()))
            assert _launches(lib) - before == 1
            got = dst.cpu().numpy()
            for f in range(F):
                blk = got[f * fs:f * fs + n * ld].reshape(n, ld)
                if feature >= 0 and f != feature:
                    np.testing.assert_array_equal(got[f * fs:(f + 1) * fs], dst0[f * fs:(f + 1) * fs])
                    continue
                keep = philox.dropout_keep(seed, step + step_dev, off + np.arange(n, dtype=np.uint64), f, layer, width,
                                           np.float32(rate))
                np.testing.assert_array_equal(blk[:, :width], R.dropout(vals[f], keep, rate).astype(np.float32))
                np.testing.assert_array_equal(blk[:, width:], dst0[f * fs:f * fs + n * ld].reshape(n, ld)[:, width:])
                np.testing.assert_array_equal(got[f * fs + n * ld:(f + 1) * fs], dst0[f * fs + n * ld:(f + 1) * fs])


# ---- reductions -------------------------------------------------------------------------------------------------------
def _ints(rng, shape):
    return rng.integers(-2000, 2000, shape).astype(np.float32)


@pytest.mark.parametrize("nrows", [0, 1, 7, 8, 9, 56, 57, 64, 65])
def test_reduce_partials_and_single_segments_are_exact(nrows):
    L_, lib = _lib()
    rng = np.random.default_rng(nrows)
    for count in (1, 31, 32, 33, 4095, 4096, 4097):
        stride = count + 5
        src = np.full((max(nrows, 1), stride), np.nan, np.float32)
        src[:nrows, :count] = _ints(rng, (nrows, count))
        ref = src[:nrows, :count].astype(np.float64).sum(0)
        S = _dev(src)
        dst = _dev(np.full(count + 4, SENTINEL, np.float32))
        before = _launches(lib)
        L_.check(lib.dib_debug_reduce(0, L_.ptr(S), stride, nrows, count, L_.ptr(dst), None, 0, None, None, 0, 0, 0, _st()))
        assert _launches(lib) - before == 1
        d = dst.cpu().numpy()
        np.testing.assert_array_equal(d[:count], ref)
        assert np.all(d[count:] == SENTINEL)
        dst2 = _dev(np.full(count + 4, SENTINEL, np.float32))
        seg = (L_.DibReduceSeg * 1)(L_.DibReduceSeg(S.data_ptr(), stride, nrows, count, 0.25, dst2.data_ptr()))
        before = _launches(lib)
        L_.check(lib.dib_debug_reduce(1, None, 0, 0, 0, None, seg, 1, None, None, 0, 0, 0, _st()))
        assert _launches(lib) - before == 1
        d2 = dst2.cpu().numpy()
        np.testing.assert_array_equal(d2[:count], ref * 0.25)
        assert np.all(d2[count:] == SENTINEL)


def test_seventeen_segments_with_empty_ones_run_once_each():
    """17 segments, count-0 ones among them (one in the first window of 8): ceil(14 live / 8) = 2 launches, and a segment
    that accumulates into its destination would show a second pass"""
    L_, lib = _lib()
    rng = np.random.default_rng(17)
    counts = [33, 0, 4096, 5, 4097, 1, 0, 31, 32, 4095, 64, 0, 7, 9000, 1, 2, 100]
    nrows = [3, 1, 8, 65, 64, 1, 2, 9, 56, 57, 0, 4, 7, 64, 1, 65, 8]
    keep, segs, refs = [], [], []
    for c, r in zip(counts, nrows):
        stride = c + 3
        src = np.full((max(r, 1), max(stride, 1)), np.nan, np.float32)
        src[:r, :c] = _ints(rng, (r, c))
        S = _dev(src)
        D = _dev(np.full(c + 2, SENTINEL, np.float32))
        keep += [S, D]
        segs.append(L_.DibReduceSeg(S.data_ptr(), stride, r, c, 2.0, D.data_ptr()))
        refs.append(src[:r, :c].astype(np.float64).sum(0) * 2.0)
    arr = (L_.DibReduceSeg * len(segs))(*segs)
    before = _launches(lib)
    L_.check(lib.dib_debug_reduce(1, None, 0, 0, 0, None, arr, len(segs), None, None, 0, 0, 0, _st()))
    live = sum(c > 0 for c in counts)
    assert _launches(lib) - before == -(-live // 8)
    for k, c in enumerate(counts):
        d = keep[2 * k + 1].cpu().numpy()
        np.testing.assert_array_equal(d[:c], refs[k])
        assert np.all(d[c:] == SENTINEL), k


@pytest.mark.parametrize("F", [1, 3, 9])
def test_finalize_stats_is_exact(F):
    L_, lib = _lib()
    rng = np.random.default_rng(F)
    for nblk_kl, nblk_loss, has_y in ((1, 1, 1), (17, 17, 1), (33, 40, 1), (5, 5, 0)):
        stride = nblk_kl + 3
        kl = np.full((F, stride), np.nan, np.float32)
        kl[:, :nblk_kl] = _ints(rng, (F, nblk_kl))
        lp = _ints(rng, nblk_loss)
        ap = _ints(rng, nblk_loss)
        out = _dev(np.full(F + 6, SENTINEL, np.float32))
        K, LP, AP = _dev(kl), _dev(lp), _dev(ap)
        before = _launches(lib)
        L_.check(lib.dib_debug_reduce(2, L_.ptr(K), stride, F, nblk_kl, L_.ptr(out), None, 0, L_.ptr(LP), L_.ptr(AP), nblk_loss,
                                      12345, has_y, _st()))
        assert _launches(lib) - before == 1
        o = out.cpu().numpy()
        np.testing.assert_array_equal(o[:F], kl[:, :nblk_kl].astype(np.float64).sum(1))
        np.testing.assert_array_equal(o[F:F + 2], [lp.sum(), ap.sum()] if has_y else [0, 0])
        assert o[F + 2] == 12345 and np.all(o[F + 3:] == SENTINEL)


# ---- public entry points: stand-alone PE, optimizers, pairwise Gaussians ----------------------------------------------
@pytest.mark.parametrize("nfreq", [1, 2, 5])
def test_positional_encoding_entry_point(nfreq):
    L_, lib = _lib()
    rng = np.random.default_rng(nfreq)
    n, d = 1000, 3
    x = rng.uniform(-1e3, 1e3, (n, d)).astype(np.float32)
    x[:3] = [[0.0, -0.0, 1e-30], [1.0, 3.14159, -2.5], [1e-3, 40.0, 160.0]]
    X = _dev(x)
    out = _dev(np.full(n * d * nfreq + 5, SENTINEL, np.float32))
    before = _launches(lib)
    L_.check(lib.dib_positional_encoding(L_.ptr(X), n, d, nfreq, L_.ptr(out), _st()))
    torch.cuda.synchronize()
    assert _launches(lib) - before == 1
    o = out.cpu().numpy()
    assert np.all(o[n * d * nfreq:] == SENTINEL)
    ref, b = R.pe_plain(x, nfreq)
    within("pe_plain", o[:n * d * nfreq].reshape(n, d * nfreq), ref, b, f"pe_plain nfreq={nfreq}")


def _opt_case(rng, count):
    w = rng.standard_normal(count + 3).astype(np.float32)
    g = rng.standard_normal(count + 3).astype(np.float32)
    g[:min(count, 5)] = 0.0                                             # g = 0
    g[5:min(count, 8)] = [1e-20, -3e4, 7.0][:max(0, min(count, 8) - 5)]
    return w, g


def _bufs(*arrs):
    return [_dev(a.copy()) for a in arrs]


@pytest.mark.parametrize("count", [0, 1, 255, 257, 1000])
def test_adam_entry_point(count):
    """steps 1 and 2 from zero moments, lr and step on the device; the step counter advances once per call, count = 0 too"""
    L_, lib = _lib()
    rng = np.random.default_rng(count)
    w, g = _opt_case(rng, count)
    z = np.zeros_like(w)
    W, G, M, V = _bufs(w, g, z, z)
    lr = _dev(np.array([1e-3], np.float32))
    step = _dev(np.array([0], np.int32))
    b1, b2, eps = 0.9, 0.999, 1e-7
    mw, mm, mv = w.astype(np.float64), z.astype(np.float64), z.astype(np.float64)
    for t in (1, 2):
        before = _launches(lib)
        L_.check(lib.dib_adam_step(L_.ptr(W), L_.ptr(G), L_.ptr(M), L_.ptr(V), count, L_.ptr(lr), L_.ptr(step), b1, b2, eps,
                                   _st()))
        torch.cuda.synchronize()
        assert _launches(lib) - before == (2 if count else 1)
        assert int(step.cpu()[0]) == t
        ref = R.adam(mw[:count], g[:count], mm[:count], mv[:count], 1e-3, t, b1, b2, eps)
        gw, gm, gv = (a.cpu().numpy() for a in (W, M, V))
        within("adam w", gw[:count], ref["w"], ref["w_bound"], f"adam count={count} t={t}")
        within("adam m", gm[:count], ref["m"], ref["m_bound"], f"adam count={count} t={t}")
        within("adam v", gv[:count], ref["v"], ref["v_bound"], f"adam count={count} t={t}")
        np.testing.assert_array_equal(gw[count:], w[count:])            # nothing past count
        mw, mm, mv = (np.concatenate([a[:count].astype(np.float64), b[count:]]) for a, b in ((gw, w), (gm, z), (gv, z)))


@pytest.mark.parametrize("count", [0, 257, 1000])
@pytest.mark.parametrize("kind,hyper", [(0, (0.0, 0.0, 0.0)), (0, (0.9, 0.0, 0.0)), (0, (0.9, 1.0, 0.0)),
                                        (1, (0.9, 0.0, 1e-7)), (1, (0.9, 0.5, 1e-7))])
def test_sgd_and_rmsprop_entry_point(count, kind, hyper):
    L_, lib = _lib()
    rng = np.random.default_rng(count + kind)
    w, g = _opt_case(rng, count)
    s1 = (rng.random(w.size) * (1.0 if kind else 0.1)).astype(np.float32)
    s2 = (rng.standard_normal(w.size) * 1e-3).astype(np.float32)
    W, G, S1, S2 = _bufs(w, g, s1, s2)
    lr = _dev(np.array([1e-2], np.float32))
    step = _dev(np.array([5], np.int32))
    before = _launches(lib)
    L_.check(lib.dib_optimizer_step(kind, L_.ptr(W), L_.ptr(G), L_.ptr(S1), L_.ptr(S2), count, L_.ptr(lr), L_.ptr(step),
                                    *hyper, _st()))
    torch.cuda.synchronize()
    assert _launches(lib) - before == (2 if count else 1)
    assert int(step.cpu()[0]) == 6
    gw, g1, g2 = (a.cpu().numpy() for a in (W, S1, S2))
    tag = f"kind={kind} hyper={hyper} count={count}"
    if kind == 0:
        ref = R.sgd(w[:count], g[:count], s1[:count], 1e-2, hyper[0], hyper[1] != 0)
        within("sgd w", gw[:count], ref["w"], ref["w_bound"], tag)
        within("sgd v", g1[:count], ref["v"], ref["v_bound"], tag)
    else:
        ref = R.rmsprop(w[:count], g[:count], s1[:count], s2[:count], 1e-2, *hyper)
        within("rmsprop w", gw[:count], ref["w"], ref["w_bound"], tag)
        within("rmsprop ms", g1[:count], ref["ms"], ref["ms_bound"], tag)
        within("rmsprop mom", g2[:count], ref["mom"], ref["mom_bound"], tag)
    for got, orig in ((gw, w), (g1, s1), (g2, s2)):
        np.testing.assert_array_equal(got[count:], orig[count:])


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("E", [1, 3, 32])
def test_pairwise_gaussian_entry_point(kind, E):
    """both kinds, la = lb exactly and within 1e-6, and a spread of variances"""
    L_, lib = _lib()
    rng = np.random.default_rng(E * 2 + kind)
    n, m = 37, 300
    ml1 = np.concatenate([rng.standard_normal((n, E)), rng.uniform(-4, 4, (n, E))], 1).astype(np.float32)
    ml2 = np.concatenate([rng.standard_normal((m, E)), rng.uniform(-4, 4, (m, E))], 1).astype(np.float32)
    ml2[:n] = ml1                                                       # identical Gaussians: D = 0
    ml2[n:2 * n, E:] = ml1[:, E:] * np.float32(1 + 1e-6)               # la ~ lb
    ml2[n:2 * n, :E] = ml1[:, :E] + np.float32(1e-3)
    A, B = _dev(ml1), _dev(ml2)
    out = _dev(np.full(n * m + 5, SENTINEL, np.float32))
    comp = _dev(np.full(n * m + 5, SENTINEL, np.float32))
    before = _launches(lib)
    L_.check(lib.dib_pairwise_gaussian(kind, L_.ptr(A), n, L_.ptr(B), m, E, L_.ptr(out), L_.ptr(comp), _st()))
    torch.cuda.synchronize()
    assert _launches(lib) - before == 1
    o, c = out.cpu().numpy(), comp.cpu().numpy()
    assert np.all(o[n * m:] == SENTINEL) and np.all(c[n * m:] == SENTINEL)
    ref = R.pairwise_gaussian(kind, ml1, ml2)
    tag = f"pairwise kind={kind} E={E}"
    within(f"pairwise{kind} D", o[:n * m].reshape(n, m), ref["D"], ref["D_bound"], tag)
    within(f"pairwise{kind} exp(-D)", c[:n * m].reshape(n, m), ref["comp"], ref["comp_bound"], tag)


def test_hooks_reject_bad_arguments():
    L_, lib = _lib()
    buf = _dev(np.zeros(64, np.float32))
    p = L_.ptr(buf)
    with pytest.raises(L_.DibError, match="ldo"):
        L_.check(lib.dib_debug_reparam(1, p, 64, 3, 1, 2, 4, None, 0, 0, None, 0, None, 1, p, 4, None, p, 1, None, None, 1.0,
                                       None, 0, _st()))
    with pytest.raises(L_.DibError, match="unknown loss"):
        L_.check(lib.dib_debug_loss(5, 0, 0.0, p, 1, p, 1, 1, 1.0, None, None, None, p, p, 0, _st()))
    with pytest.raises(L_.DibError, match="kind"):
        L_.check(lib.dib_debug_reduce(3, None, 0, 0, 0, None, None, 0, None, None, 0, 0, 0, _st()))
    with pytest.raises(L_.DibError, match="rate"):
        L_.check(lib.dib_debug_dropout(p, p, 8, 2, 2, 1, 1, 1.0, 0, 0, None, 0, 0, -1, 0, 0, _st()))


def test_zz_report_worst_ratios():
    for k in sorted(WORST):
        print(f"[elementwise] worst measured / bound {k}: {WORST[k]:.3g}")
