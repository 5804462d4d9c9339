"""GPU (H100): the InfoNCE kernels element by element against the float64 reference with per-element bounds
(tests/infonce_stream_reference.py).  The streaming sweeps run through dib_debug_infonce_stream, which launches them as the
training step does; the materialised head runs through utils.infonce_loss_and_grads.  Every case also checks the sweeps'
memory contracts: NaN in every input element they must not read, a sentinel in every output element they must not write."""
import ctypes

import numpy as np
import pytest
import torch

from tests import infonce_stream_reference as R
from tests.fp_exact import C_BOUND, U, round_tf32, within
from tests.gpu_cases import _dev, _lib

pytestmark = pytest.mark.gpu

KIND = {k: i for i, k in enumerate(R.KINDS)}
SENTINEL = np.float32(-3.0e33)
WORST = {}


def padded_input(e, ld):
    """[n, d] -> device [32 ceil(n / 32) + 32, ld] with NaN in the pad columns and in every row past n."""
    n, d = e.shape
    buf = np.full((-(-n // 32) * 32 + 32, ld), np.nan, np.float32)
    buf[:n, :d] = e
    return _dev(buf)


def sentinel(*shape):
    return _dev(np.full(shape, SENTINEL, np.float32))


def stream(kind, T, e1, e2, parts=None, phases=3, lse_stride=1, round_out=0, lse_in=None, sides=(True, True)):
    """Run the sweeps over the row ranges `parts` (default: all rows): the loss sweeps of every part, then the gradient sweeps of
    every part, as data-parallel ranks do.  Checks the memory contracts and the launch count; returns the outputs as numpy."""
    L, lib = _lib()
    n, d = e1.shape
    ld1, ld2, ldo = d + 3, d + 8, d + 5
    E1, E2 = padded_input(e1, ld1), padded_input(e2, ld2)
    parts = parts or [(0, n)]
    lr, lc = sentinel(n * lse_stride + 40), sentinel(n * lse_stride + 40)
    if lse_in is not None:
        lr[:n * lse_stride:lse_stride] = _dev(np.asarray(lse_in[0], np.float32))
        lc[:n * lse_stride:lse_stride] = _dev(np.asarray(lse_in[1], np.float32))
    bufs = [dict(diag=sentinel(rows + 33), loss=sentinel(4), d1=sentinel(rows + 2, ldo) if sides[0] else None,
                 d2=sentinel(rows + 2, ldo) if sides[1] else None) for _, rows in parts]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = L.ptr
    for phase in (1, 2):
        if not phases & phase:
            continue
        for (row0, rows), b in zip(parts, bufs):
            before = int(lib.dib_launch_count())
            L.check(lib.dib_debug_infonce_stream(KIND[kind], float(T), p(E1), ld1, p(E2), ld2, n, d, row0, rows, p(lr), p(lc),
                                                 lse_stride, p(b["diag"]), p(b["loss"]), p(b["d1"]), ldo, p(b["d2"]), ldo,
                                                 round_out, phase, st))
            assert int(lib.dib_launch_count()) - before == (3 if phase == 1 else sum(sides))
    out = {}
    for name, buf in (("r", lr), ("c", lc)):
        v = buf.cpu().numpy()
        written = np.zeros(v.shape, bool)
        idx = np.arange(n) * lse_stride
        if phases & 1 and lse_in is None:
            for row0, rows in parts:
                written[idx[row0:row0 + rows]] = True
        else:
            written[idx] = True
        assert np.all(v[~written] == SENTINEL), f"{name}: an element outside the own rows' slots was written"
        out[name] = v[idx].astype(np.float64)
    for key in ("diag", "d1", "d2"):
        chunks = []
        for (row0, rows), b in zip(parts, bufs):
            if b.get(key) is None:
                continue
            v = b[key].cpu().numpy()
            if key == "diag" and not phases & 1:
                assert np.all(v == SENTINEL)
                continue
            if key != "diag" and not phases & 2:
                assert np.all(v == SENTINEL)
                continue
            assert np.all(v[rows:] == SENTINEL), f"{key}: a row past the own rows was written"
            if key != "diag":
                assert np.all(v[:rows, d:] == 0.0), f"{key}: pad columns [d, ld) not zeroed"
                v = v[:rows, :d]
            else:
                v = v[:rows]
            chunks.append(v)
        if chunks:
            out[key] = np.concatenate(chunks).astype(np.float64)
    if phases & 1:
        losses = [b["loss"].cpu().numpy() for b in bufs]
        for v in losses:
            assert np.all(v[1:] == SENTINEL)
        out["loss"] = [float(v[0]) for v in losses]
    return out


def check_stream(kind, T, e1, e2, ref, tag, grads=True):
    out = stream(kind, T, e1, e2, phases=3 if grads else 1)
    within(WORST, "r", out["r"], ref["r"], C_BOUND * ref["rho_r"], tag)
    within(WORST, "c", out["c"], ref["c"], C_BOUND * ref["rho_c"], tag)
    within(WORST, "s_ii", out["diag"], ref["diag"], C_BOUND * ref["sigma_diag"], tag)
    within(WORST, "loss_sum", out["loss"][0], ref["loss"], ref["loss_bound"], tag)
    if grads:
        within(WORST, "d_e1", out["d1"], ref["d1"], ref["d1_bound"], tag)
        within(WORST, "d_e2", out["d2"], ref["d2"], ref["d2_bound"], tag)
    return out


# every (n, d) of the shape list at the normal regime, for all five similarities
@pytest.mark.parametrize("n,d", R.GRAD_SHAPES)
@pytest.mark.parametrize("kind", R.KINDS)
def test_stream_shapes(kind, n, d):
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=11)
    ref = R.reference(e1, e2, kind, T)
    out = check_stream(kind, T, e1, e2, ref, f"{kind} n={n} d={d}")
    if n == 1:
        assert out["loss"][0] == 0.0 and np.all(out["d1"] == 0.0) and np.all(out["d2"] == 0.0)


@pytest.mark.parametrize("regime,T", [("wide", 2.0 ** -8), ("wide", 1.0), ("wide", 2.0 ** 8), ("peaked", 1.0),
                                      ("identical", 1.0), ("duplicate", 1.0), ("dyadic", 1.0), ("dyadic", 2.0 ** -8)])
@pytest.mark.parametrize("n,d", [(33, 31), (100, 3), (65, 257)])
@pytest.mark.parametrize("kind", R.KINDS)
def test_stream_regimes(kind, n, d, regime, T):
    e1, e2, T = R.case_data(kind, n, d, regime, T=T, seed=12)
    ref = R.reference(e1, e2, kind, T)
    if regime == "wide" and (kind != "cosine" or T < 1):
        P = R.Pairs(e1, e2, kind, T)
        assert (P.s.max(1) - P.s.min(1)).max() > 200
    out = check_stream(kind, T, e1, e2, ref, f"{kind} {regime} T={T} n={n} d={d}")
    if regime == "dyadic" and kind in ("l2sq", "l1", "linf"):
        np.testing.assert_array_equal(out["diag"], ref["diag"])          # sigma = 0: the kernels' s_ii is exact


@pytest.mark.parametrize("kind", ["l2", "cosine"])
def test_stream_large_ragged_n_loss_sweeps(kind):
    n, d = 20001, 2
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=13)
    ref = R.reference(e1, e2, kind, T, grads=False)
    check_stream(kind, T, e1, e2, ref, f"{kind} n={n} d={d}", grads=False)


@pytest.mark.parametrize("kind", R.KINDS)
def test_gradient_sweeps_alone_from_float64_log_sum_exps(kind):
    """Phase 2 alone, fed the float64 r and c rounded to fp32 (rho = their rounding): the gradient sweep in isolation."""
    n, d = 100, 33
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=14)
    lse = R.log_sum_exps(e1, e2, kind, T)
    r32, c32 = lse["r"].astype(np.float32), lse["c"].astype(np.float32)
    rho_r = np.abs(r32 - lse["r"]) + U * np.abs(lse["r"])
    rho_c = np.abs(c32 - lse["c"]) + U * np.abs(lse["c"])
    out = stream(kind, T, e1, e2, phases=2, lse_in=(r32, c32))
    g1, b1 = R.side_gradient(e1, e2, kind, T, lse["r"], lse["c"], rho_r, rho_c)
    g2, b2 = R.side_gradient(e2, e1, kind, T, lse["c"], lse["r"], rho_c, rho_r)
    within(WORST, "d_e1 (phase 2)", out["d1"], g1, b1, kind)
    within(WORST, "d_e2 (phase 2)", out["d2"], g2, b2, kind)


@pytest.mark.parametrize("kind", R.KINDS)
def test_uneven_partitions_repeat_strides_and_round_out(kind):
    """Uneven row ranges reproduce every per-row output of the full-range call bit for bit; repeated calls are bit-identical;
    r / c at lse_stride 2 leave the other slot alone; round_out = 1 gives the TF32 rounding of the round_out = 0 gradients;
    s_ii equals the diagonal of dib_scaled_similarity."""
    from dib_b200 import utils
    n, d = 100, 33
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=15)
    full = stream(kind, T, e1, e2)
    again = stream(kind, T, e1, e2)
    for k in ("r", "c", "diag", "d1", "d2", "loss"):
        np.testing.assert_array_equal(full[k], again[k], err_msg=k)
    split = stream(kind, T, e1, e2, parts=[(0, 1), (1, 32), (33, n - 33)], lse_stride=2)
    for k in ("r", "c", "diag", "d1", "d2"):
        np.testing.assert_array_equal(split[k], full[k], err_msg=k)
    rounded = stream(kind, T, e1, e2, round_out=1, sides=(False, True))
    assert "d1" not in rounded
    np.testing.assert_array_equal(rounded["d2"], round_tf32(full["d2"].astype(np.float32)))
    S = utils.get_scaled_similarity(torch.from_numpy(e1).cuda(), torch.from_numpy(e2).cuda(), kind, T).cpu().numpy()
    np.testing.assert_array_equal(np.diag(S).astype(np.float64), full["diag"])


def test_cosine_at_d1_has_an_exactly_zero_gradient():
    rng = np.random.default_rng(16)
    n = 45
    e1 = (rng.choice([-1, 1], (n, 1)) * 2.0 ** rng.integers(-3, 4, (n, 1))).astype(np.float32)
    e2 = (rng.choice([-1, 1], (n, 1)) * 2.0 ** rng.integers(-3, 4, (n, 1))).astype(np.float32)
    out = stream("cosine", 0.5, e1, e2)
    assert np.all(out["d1"] == 0.0) and np.all(out["d2"] == 0.0)


def test_hook_rejects_what_the_library_cannot_run():
    L, lib = _lib()
    e = torch.zeros(64, 600, device="cuda")
    buf = torch.zeros(4096, device="cuda")
    p, st = L.ptr, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(kind=0, T=1.0, ld=8, n=10, d=8, row0=0, rows=10, stride=1, phases=3):
        return lib.dib_debug_infonce_stream(kind, T, p(e), ld, p(e), ld, n, d, row0, rows, p(buf), p(buf), stride, p(buf),
                                            p(buf), p(buf), ld, p(buf), ld, 0, phases, st)
    for bad in (dict(d=0), dict(d=513, ld=513), dict(ld=7), dict(T=0.0), dict(T=-1.0), dict(T=float("inf")), dict(kind=5),
                dict(row0=5, rows=6), dict(rows=0), dict(row0=-1), dict(stride=0), dict(phases=0), dict(phases=4), dict(n=0)):
        assert call(**bad) != 0, bad
        assert lib.dib_last_error().startswith(b"dib_debug_infonce_stream"), lib.dib_last_error()
    assert call() == 0


@pytest.mark.parametrize("n,d", [(1, 3), (31, 33), (33, 1), (33, 512), (300, 31), (300, 257), (1000, 2), (1000, 64)])
@pytest.mark.parametrize("kind", R.KINDS)
def test_materialised_head(kind, n, d):
    from dib_b200 import utils
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=17)
    ref = R.reference(e1, e2, kind, T, head=True)
    loss, d1, d2 = utils.infonce_loss_and_grads(torch.from_numpy(e1).cuda(), torch.from_numpy(e2).cuda(), kind, T)
    tag = f"head {kind} n={n} d={d}"
    within(WORST, "head loss", loss.item(), ref["loss"] / n, ref["loss_bound"] / n + C_BOUND * U * abs(ref["loss"] / n), tag)
    within(WORST, "head d_e1", d1.cpu().numpy(), ref["d1"], ref["d1_bound"], tag)
    within(WORST, "head d_e2", d2.cpu().numpy(), ref["d2"], ref["d2_bound"], tag)


@pytest.mark.parametrize("kind", ["l2sq", "l1", "linf"])
def test_materialised_head_on_dyadic_ties(kind):
    from dib_b200 import utils
    n, d = 33, 31
    e1, e2, T = R.case_data(kind, n, d, "dyadic", seed=18)
    ref = R.reference(e1, e2, kind, T, head=True)
    _, d1, d2 = utils.infonce_loss_and_grads(torch.from_numpy(e1).cuda(), torch.from_numpy(e2).cuda(), kind, T)
    within(WORST, "head d_e1", d1.cpu().numpy(), ref["d1"], ref["d1_bound"], f"head {kind} dyadic")
    within(WORST, "head d_e2", d2.cpu().numpy(), ref["d2"], ref["d2_bound"], f"head {kind} dyadic")


def test_zz_print_worst_ratios():
    print("worst measured / bound over the file:", {k: round(v, 4) for k, v in sorted(WORST.items())})
