"""GPU (H100): the grouped dense-layer GEMM kernels -- dib_gemm_simt.cu (exact fp32 FMA) and dib_gemm_tc.cu (tf32 wgmma) --
launched through dib_debug_gemm exactly as the library's steps launch them, against the float64 reference of
tests/grouped_gemm_reference.py, bit for bit.

Exact operands: every A / B / bias entry is i / 4 with |i| <= 4 and every DGRAD activation source is k / 16 in (-1, 1).
With reductions of at most 512 terms every product, every partial sum in any order and every o * act'(x) then fits in 24
significant bits, and every operand is exact in tf32, so both kernels must equal the float64 result exactly.  The
reference rounds only where the kernels round: one fp32 rounding of alpha * z (leaky ReLU FWD) and of o * alpha (leaky
ReLU DGRAD), and cvt.rna.tf32 under round_out.  tanh / sigmoid / elu in FWD (libdevice) are the one inexact case and are
held to a ulp bound instead.

Every float the kernels must not read is NaN (rows at or beyond M, W rows at or beyond T, the slab tails between
problems); every float they must not write holds a sentinel (outside [R x ldc], other problems' regions, outside each
split's partial slice).  The whole output buffer is compared, so a missed, doubled or stray write fails.

The end of the file runs the generic (non-fused) training path at the model level: a group whose weight-gradient grid
exceeds 65 535 slices, row isolation across the weight-gradient batch splits, and one handle stepping through different
split counts."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests.fp_exact import dyadic, fits, round_tf32
from tests.fused16_oracle import per_variable_errors
from tests.gpu_cases import _L, build_model, rel_err
from tests.grouped_gemm_reference import INEXACT_ACTS, act_source, assert_on_grid, ref_dgrad, ref_fwd, ref_wgrad, ulp32

pytestmark = pytest.mark.gpu

FWD, DGRAD, WGRAD = 0, 1, 2
ACTS = {"linear": 0, "relu": 1, "tanh": 2, "leaky_relu": 3, "sigmoid": 4, "elu": 5}
SENTINEL = np.float32(-7777.25)


# ---------------------------------------------------------------------------------------------------------------------
# one grouped launch: buffers laid out as dib_api.cu's make_buf lays them out, with NaN and sentinel moats
# ---------------------------------------------------------------------------------------------------------------------
def _ru(v, m):
    return (v + m - 1) // m * m


class Group:
    """nprob problems of one mode.  T / C / R: per-problem lists.  Every problem owns a slab of `rows * ld` floats of each
    activation-like operand, at a feature stride rounded to 64 floats (make_buf); the parameters are W then bias per
    problem at a fixed stride, with NaN gaps behind each."""

    def __init__(self, mode, T, C, R=None, M=1, act="linear", alpha=0.2, round_out=0, nsplit=1, rps=0, seed=0,
                 ld_round=4, extra_rows=3, bias_apart=False):
        self.mode, self.T, self.C, self.R = mode, list(T), list(C), list(R) if R is not None else [0] * len(T)
        self.n = len(self.T)
        self.M, self.act, self.alpha, self.round_out = M, act, float(alpha), int(round_out)
        self.nsplit, self.rps = nsplit, rps
        rng = np.random.default_rng(seed)
        Ma = M + extra_rows                                   # rows at or beyond M stay NaN: never read
        n = self.n
        probs = (_L().DibGemmProblem * n)()
        self.probs = probs
        if mode in (FWD, DGRAD):
            # A: [M x lda] activations (FWD: T = fan-in) or output gradients (DGRAD: T = fan-out)
            lda = [_ru(t, ld_round) for t in self.T]
            ldc = [_ru(c, 4) for c in self.C]
            fsA, fsC = _ru(Ma * max(lda), 64), _ru(Ma * max(ldc), 64)
            A = np.full(fsA * n + 64, np.nan, np.float32)
            Cbuf = np.full(fsC * n + 64, SENTINEL, np.float32)
            X = np.full(fsC * n + 64, np.nan, np.float32)
            # parameters: W [T x C] (FWD) or [C x T] (DGRAD) with ldb = its column count, then bias [C]
            wrows = [t if mode == FWD else c for t, c in zip(self.T, self.C)]
            ldb = [c if mode == FWD else t for t, c in zip(self.T, self.C)]
            wsz = max(r * l for r, l in zip(wrows, ldb))
            bias_at = _ru(wsz + 2 * max(ldb), 4)              # two NaN rows behind W: rows at or beyond T are not read
            pstride = _ru(bias_at + max(self.C) + 8, 4)
            P = np.full(pstride * n + 64, np.nan, np.float32)
            self.a, self.w, self.b, self.x = [], [], [], []
            for g in range(n):
                T_, C_ = self.T[g], self.C[g]
                a = dyadic(rng, (M, T_), dtype=np.float32)
                blk = np.zeros((Ma, lda[g]), np.float32)
                blk[M:] = np.nan
                blk[:M, :T_] = a                              # pad columns are zeros (the buffers' invariant)
                A[g * fsA:g * fsA + Ma * lda[g]] = blk.ravel()
                w = dyadic(rng, (wrows[g], ldb[g]), dtype=np.float32)
                P[g * pstride:g * pstride + w.size] = w.ravel()
                b = dyadic(rng, (C_,), dtype=np.float32)
                if mode == FWD:
                    P[g * pstride + bias_at:g * pstride + bias_at + C_] = b
                x = act_source(rng, (M, C_))
                xb = np.zeros((Ma, ldc[g]), np.float32)
                xb[M:] = np.nan
                xb[:M, :C_] = x
                X[g * fsC:g * fsC + Ma * ldc[g]] = xb.ravel()
                self.a.append(a); self.w.append(w); self.b.append(b); self.x.append(x)
                p = probs[g]
                p.a_off, p.lda = g * fsA, lda[g]
                p.b_off, p.ldb = g * pstride, ldb[g]
                p.c_off, p.ldc = g * fsC, ldc[g]
                p.x_off = g * pstride + bias_at if mode == FWD else g * fsC
                p.ldx = ldc[g] if mode == DGRAD else 0
                p.T, p.C, p.R, p.act = T_, C_, 0, ACTS[act]
            self.host = {"A": A, "B": P, "C": Cbuf, "X": X}
            self.fsC, self.ldc = fsC, ldc
            if bias_apart:
                # the tensor-core launches of the library read W from the tf32 weight shadow and the bias from the
                # parameters: here a W-only copy and a bias-only copy, each NaN where the other holds the values
                Wonly, Bonly = P.copy(), np.full_like(P, np.nan)
                for g in range(n):
                    o = g * pstride + bias_at
                    Bonly[o:o + self.C[g]] = P[o:o + self.C[g]]
                    Wonly[o:o + self.C[g]] = np.nan
                self.host["B"], self.host["bias"] = Wonly, Bonly
        else:
            # WGRAD: A = h [M x lda] (R = fan-in), B = dz [M x ldb] (C = fan-out); partials [R x C] then bias [C] per
            # problem inside each split's slice of split_stride floats
            lda = [_ru(r, ld_round) for r in self.R]
            ldb = [_ru(c, ld_round) for c in self.C]
            fsA, fsB = _ru(Ma * max(lda), 64), _ru(Ma * max(ldb), 64)
            A = np.full(fsA * n + 64, np.nan, np.float32)
            B = np.full(fsB * n + 64, np.nan, np.float32)
            dwsz = max(r * c for r, c in zip(self.R, self.C))
            db_at = _ru(dwsz + 4, 4)                         # a sentinel gap between dW and db
            pstride = _ru(db_at + max(self.C) + 4, 4)
            self.split_stride = _ru(pstride * n + 8, 64)
            Cbuf = np.full(self.split_stride * nsplit + 64, SENTINEL, np.float32)
            self.h, self.dz = [], []
            for g in range(n):
                R_, C_ = self.R[g], self.C[g]
                h = dyadic(rng, (M, R_), dtype=np.float32)
                dz = dyadic(rng, (M, C_), dtype=np.float32)
                for buf, v, ld, fs in ((A, h, lda[g], fsA), (B, dz, ldb[g], fsB)):
                    blk = np.zeros((Ma, ld), np.float32)
                    blk[M:] = np.nan
                    blk[:M, :v.shape[1]] = v
                    buf[g * fs:g * fs + Ma * ld] = blk.ravel()
                self.h.append(h); self.dz.append(dz)
                p = probs[g]
                p.a_off, p.lda = g * fsA, lda[g]
                p.b_off, p.ldb = g * fsB, ldb[g]
                p.c_off, p.ldc = g * pstride, C_
                p.x_off, p.ldx = g * pstride + db_at, 0
                p.T, p.C, p.R, p.act = 0, C_, R_, 0
            self.host = {"A": A, "B": B, "C": Cbuf}
            self.pstride = pstride

    def expected(self):
        """(the whole expected output buffer, mask of the floats the kernels write).  Inexact activations: the float64
        values in a separate array at the written positions."""
        exp = self.host["C"].copy()
        exp64 = exp.astype(np.float64)
        mask = np.zeros(exp.shape, bool)
        M = self.M
        if self.mode in (FWD, DGRAD):
            for g in range(self.n):
                C_, ldc = self.C[g], self.ldc[g]
                if self.mode == FWD:
                    v = ref_fwd(self.a[g], self.w[g], self.b[g], self.act, self.alpha, self.round_out)
                else:
                    v = ref_dgrad(self.a[g], self.w[g], self.x[g], self.act, self.alpha, self.round_out)
                blk = np.zeros((M, ldc), np.float64)            # pad columns up to ldc are written as zeros
                blk[:, :C_] = v
                o = g * self.fsC
                exp64[o:o + M * ldc] = blk.ravel()
                exp[o:o + M * ldc] = blk.ravel().astype(np.float32)
                mask[o:o + M * ldc] = True
        else:
            for g in range(self.n):
                R_, C_ = self.R[g], self.C[g]
                dw, db = ref_wgrad(self.h[g], self.dz[g], M, self.nsplit, self.rps)
                p = self.probs[g]
                for s in range(self.nsplit):
                    o = s * self.split_stride + p.c_off
                    exp[o:o + R_ * C_] = dw[s].ravel(); mask[o:o + R_ * C_] = True
                    o = s * self.split_stride + p.x_off
                    exp[o:o + C_] = db[s]; mask[o:o + C_] = True
            exp64 = exp.astype(np.float64)
        return exp, exp64, mask

    def launch(self, kernel, chunks=1):
        """Run the group on `kernel` ('simt' | 'tc'); returns the output buffer.  Asserts the launch count: one launch, or
        `chunks` when the group's grid needs several."""
        lib = _L().load()
        dev = torch.device("cuda")
        d = {k: torch.from_numpy(v).to(dev) for k, v in self.host.items()}
        bias = d.get("bias", d["B"])
        X = d["C"] if self.mode == WGRAD else d["X"]
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        maxC, maxR = max(self.C), max(self.R)
        before = int(lib.dib_launch_count())
        rc = lib.dib_debug_gemm(_L().GEMM_KERNELS[kernel], self.mode, ctypes.cast(self.probs, ctypes.c_void_p), self.n, _L().ptr(d["A"]),
                                _L().ptr(d["B"]), _L().ptr(d["C"]), _L().ptr(X), _L().ptr(bias), self.M, maxC, maxR,
                                self.nsplit, self.rps, getattr(self, "split_stride", 0), self.alpha, self.round_out, st)
        _L().check(rc)
        launches = int(lib.dib_launch_count()) - before
        assert launches == chunks, (kernel, launches, chunks)
        return d["C"].cpu().numpy()


# worst errors of the inexact FWD epilogues seen in this process: (act, round_out) -> fp32 ulps (tf32 ulps under round_out)
_WORST = {}
# Bound: 3 fp32 ulps of the float64 value, plus one tf32 ulp under round_out.  Measured on an H100 80GB HBM3 (700 W):
# tanh 1.27, sigmoid 1.60, elu 0.77 fp32 ulps; under round_out 0.50 tf32 ulps.
INEXACT_ULPS = 3


def check(group, got):
    exp, exp64, mask = group.expected()
    assert np.isfinite(got).all(), "non-finite output (a NaN operand was read)"
    if group.mode == FWD and group.act in INEXACT_ACTS:
        assert np.array_equal(got[~mask], exp[~mask]), "a float outside the output regions was written"
        g, r = got[mask].astype(np.float64), exp64[mask]
        unit = ulp32(r)
        if group.round_out:
            err = np.abs(g - r) / (unit * 2.0 ** 13)
            assert np.all(np.abs(g - r) <= INEXACT_ULPS * unit + unit * 2.0 ** 13), float(err.max())
            assert np.array_equal(round_tf32(got[mask]), got[mask]), "round_out: outputs off the tf32 grid"
        else:
            err = np.abs(g - r) / unit
            assert err.max() <= INEXACT_ULPS, float(err.max())
        key = (group.act, group.round_out)
        _WORST[key] = max(_WORST.get(key, 0.0), float(err.max()))
        return
    if not np.array_equal(got, exp):
        bad = np.flatnonzero(got != exp)
        where = "inside" if mask[bad[0]] else "outside"
        raise AssertionError(f"{bad.size} floats differ, first at {bad[0]} ({where} the written region): "
                             f"got {got[bad[0]]}, want {exp[bad[0]]}")


def tc_eligible(mode, T, C, R=0, ld_round=4):
    """dib_gemm_tc_eligible's rule for a uniform group laid out by Group."""
    if C % 64:
        return False
    if mode == FWD:
        return T >= 32 and _ru(T, ld_round) >= 32
    if mode == DGRAD:
        return T >= 32 and T % 4 == 0
    return _ru(R, ld_round) % 32 == 0 and _ru(C, ld_round) % 32 == 0


# ---------------------------------------------------------------------------------------------------------------------
# 1. every activation in FWD and DGRAD, both round_out values, alpha 0.25 and 0.2
# ---------------------------------------------------------------------------------------------------------------------
ACT_CASES = [(a, al) for a in ACTS for al in ((0.25, 0.2) if a == "leaky_relu" else (0.2,))]


@pytest.mark.parametrize("kernel", ["simt", "tc"])
@pytest.mark.parametrize("mode", [FWD, DGRAD])
@pytest.mark.parametrize("act,alpha", ACT_CASES)
@pytest.mark.parametrize("round_out", [0, 1])
def test_epilogues(kernel, mode, act, alpha, round_out):
    T = 95 if mode == FWD else 100                    # ragged against every K step; DGRAD tc needs T % 4 == 0
    g = Group(mode, [T] * 3, [128] * 3, M=129, act=act, alpha=alpha, round_out=round_out, seed=10 * mode + list(ACTS).index(act))
    assert tc_eligible(mode, T, 128)
    check(g, g.launch(kernel))


# ---------------------------------------------------------------------------------------------------------------------
# 2. FWD / DGRAD: batch rows, K ragged against the pipeline, both tc tile widths, the simt tile configurations
# ---------------------------------------------------------------------------------------------------------------------
TC_T = {FWD: [32, 33, 95, 160, 289, 512], DGRAD: [32, 36, 100, 160, 292, 512]}    # 1, 2, 3 (4), 5, 10, 16 K tiles


@pytest.mark.parametrize("mode", [FWD, DGRAD])
@pytest.mark.parametrize("M", [1, 127, 128, 129, 4097])
@pytest.mark.parametrize("kernel", ["simt", "tc"])
def test_rows_and_k_tiles(mode, M, kernel):
    """Every T of TC_T at C = 128 (tc BN = 128) and C = 192 (C % 128 = 64: BN = 64), leaky ReLU with alpha 0.25."""
    for i, T in enumerate(TC_T[mode]):
        for C in (128, 192):
            if M == 4097 and C == 192 and T not in (33, 36, 512):
                continue
            g = Group(mode, [T] * 3, [C] * 3, M=M, act="leaky_relu", alpha=0.25, round_out=i % 2, seed=M + T + C)
            assert tc_eligible(mode, T, C)
            check(g, g.launch(kernel))


@pytest.mark.parametrize("mode", [FWD, DGRAD])
@pytest.mark.parametrize("C", [1, 3, 16, 17, 33, 64, 65, 100, 130])
def test_simt_tiles_and_pad_columns(mode, C):
    """The three simt FWD / DGRAD configurations (C <= 16, 17..64, > 64), C not a multiple of 4 (pad columns up to ldc
    written as zeros), T = 1, 3 and T ragged against BT = 8 / 16."""
    for T in (1, 3, 8, 17, 33):
        for M in (1, 129, 300):
            g = Group(mode, [T] * 2, [C] * 2, M=M, act="relu", seed=T * 7 + C + M)
            check(g, g.launch("simt"))


def test_tc_refuses_what_it_cannot_run():
    """The tc choice never falls back: a group the tensor-core kernel cannot run is an error with a message."""
    for mode, T, C in ((FWD, 96, 100), (FWD, 8, 128), (DGRAD, 33, 128), (DGRAD, 96, 96)):
        g = Group(mode, [T] * 2, [C] * 2, M=64)
        assert not tc_eligible(mode, T, C)
        with pytest.raises(_L().DibError, match="tensor-core kernel cannot run"):
            g.launch("tc")
        check(g, g.launch("simt"))
    g = Group(FWD, [40, 48], [128, 128], M=64)        # heterogeneous T
    with pytest.raises(_L().DibError, match="tensor-core kernel cannot run"):
        g.launch("tc")


# ---------------------------------------------------------------------------------------------------------------------
# 3. WGRAD: the split partials
# ---------------------------------------------------------------------------------------------------------------------
def _splits(M, rps, extra=0):
    return max(math.ceil(M / rps), 1) + extra


@pytest.mark.parametrize("M,rps,extra", [(1, 64, 0), (128, 64, 1), (129, 64, 0), (4097, 256, 0), (4097, 256, 2),
                                         (2000, 512, 0), (7937 + 64, 256, 0)])
@pytest.mark.parametrize("R,C", [(1, 3), (5, 64), (32, 65), (32, 128), (33, 16), (40, 17), (128, 64), (130, 130)])
def test_wgrad_simt(M, rps, extra, R, C):
    """The five simt WGRAD configurations (R <= 32 with C > 64 / <= 64; R > 32 with C > 64, 17..64, <= 16), splits of
    whole 64-row blocks with a short last split, and splits past the batch (t_begin >= M) that must write zero partials."""
    g = Group(WGRAD, [0] * 3, [C] * 3, [R] * 3, M=M, nsplit=_splits(M, rps, extra), rps=rps, seed=M + R * 3 + C)
    check(g, g.launch("simt"))


@pytest.mark.parametrize("M,rps,extra", [(1, 64, 0), (128, 64, 1), (129, 64, 0), (4097, 256, 0), (4097, 256, 2),
                                         (2000, 512, 0)])
@pytest.mark.parametrize("R,C", [(32, 64), (128, 128), (160, 192), (40, 128)])
def test_wgrad_tc(M, rps, extra, R, C):
    """Both tc tile widths; R = 40 pads h to lda = 64 (zeros); 64-row splits are two K tiles, 512-row splits wrap the
    4-stage ring four times."""
    g = Group(WGRAD, [0] * 3, [C] * 3, [R] * 3, M=M, nsplit=_splits(M, rps, extra), rps=rps, seed=M + R + C, ld_round=32)
    assert tc_eligible(WGRAD, 0, C, R, ld_round=32)
    check(g, g.launch("tc"))
    check(g, g.launch("simt"))


# ---------------------------------------------------------------------------------------------------------------------
# 4. grouped launches
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nprob", [1, 3, 140])
@pytest.mark.parametrize("kernel", ["simt", "tc"])
def test_groups(nprob, kernel):
    """A single problem, a few and many at make_buf's feature strides, in every mode."""
    M = 129
    for mode, T in ((FWD, 33), (DGRAD, 36)):
        g = Group(mode, [T] * nprob, [64] * nprob, M=M, act="elu" if mode == DGRAD else "relu", round_out=1, seed=nprob)
        check(g, g.launch(kernel))
    g = Group(WGRAD, [0] * nprob, [64] * nprob, [96] * nprob, M=M, nsplit=3, rps=64, seed=nprob, ld_round=32)
    check(g, g.launch(kernel))


def test_tc_fwd_reads_bias_from_its_own_base():
    """As the library launches tf32 FWD (W from the tf32 shadow, bias from the parameters): NaN in the other copy."""
    for C in (64, 128):
        g = Group(FWD, [64] * 3, [C] * 3, M=130, act="leaky_relu", alpha=0.2, round_out=1, bias_apart=True, seed=C)
        check(g, g.launch("tc"))


def test_simt_heterogeneous_group():
    """Different T / C / R per problem under one maxC / maxR, as heterogeneous feature dimensionalities produce."""
    T, C, R = [10, 5, 10, 5, 3], [128, 128, 100, 17, 64], [10, 5, 40, 5, 33]
    for act in ("relu", "tanh"):
        g = Group(FWD, T, C, M=300, act=act, seed=1)
        check(g, g.launch("simt"))
        g = Group(DGRAD, C, T, M=300, act=act, seed=2)
        check(g, g.launch("simt"))
    g = Group(WGRAD, [0] * 5, C, R, M=1000, nsplit=4, rps=256, seed=3)
    check(g, g.launch("simt"))
    g = Group(WGRAD, [0] * 5, [12, 3, 17, 40, 8], [30, 2, 17, 20, 32], M=1000, nsplit=4, rps=256, seed=4)
    check(g, g.launch("simt"))


# ---------------------------------------------------------------------------------------------------------------------
# 5. groups whose grid exceeds 65 535 slices along z: consecutive launches over the problems
# ---------------------------------------------------------------------------------------------------------------------
def test_wgrad_group_over_the_grid_limit():
    """1 100 problems x 60 splits of 64 rows = 66 000 > 65 535 grid slices: two launches of 1 092 and 8 problems on both
    kernels (the tc one builds the second launch's TMA maps from its own first descriptor); a group that fits takes one."""
    n, ns, rps, R, C = 1100, 60, 64, 32, 64
    M = ns * rps
    g = Group(WGRAD, [0] * n, [C] * n, [R] * n, M=M, nsplit=ns, rps=rps, seed=5, ld_round=32, extra_rows=0)
    exp = _wgrad_expected_batched(g)
    for kernel in ("tc", "simt"):
        got = g.launch(kernel, chunks=2)
        assert np.array_equal(got, exp), (kernel, int(np.count_nonzero(got != exp)))
    # the first 1 092 problems alone: 65 520 slices, one launch; the other problems' regions keep the sentinel
    for q in range(1092, n):
        p = g.probs[q]
        for s in range(ns):
            o = s * g.split_stride
            exp[o + p.c_off:o + p.c_off + R * C] = SENTINEL
            exp[o + p.x_off:o + p.x_off + C] = SENTINEL
    g.n = 1092
    for kernel in ("tc", "simt"):
        got = g.launch(kernel, chunks=1)
        assert np.array_equal(got, exp), (kernel, int(np.count_nonzero(got != exp)))


def _wgrad_expected_batched(g):
    """Group.expected for a large uniform WGRAD group: batched float64 contractions over blocks of problems."""
    n, ns, rps, R, C = g.n, g.nsplit, g.rps, g.R[0], g.C[0]
    fits(np.array([rps * 16]), 1.0, "WGRAD sums")        # |h|, |dz| <= 1: every sum is below rps in magnitude
    exp = g.host["C"].copy()
    for q0 in range(0, n, 64):
        q1 = min(n, q0 + 64)
        h = np.stack(g.h[q0:q1]).astype(np.float64).reshape(q1 - q0, ns, rps, R)
        dz = np.stack(g.dz[q0:q1]).astype(np.float64).reshape(q1 - q0, ns, rps, C)
        assert_on_grid(h, 4); assert_on_grid(dz, 4)
        dw = np.matmul(h.transpose(0, 1, 3, 2), dz).astype(np.float32)      # [problems, ns, R, C]
        db = dz.sum(2).astype(np.float32)                                   # [problems, ns, C]
        for q in range(q0, q1):
            p = g.probs[q]
            for s in range(ns):
                o = s * g.split_stride
                exp[o + p.c_off:o + p.c_off + R * C] = dw[q - q0, s].ravel()
                exp[o + p.x_off:o + p.x_off + C] = db[q - q0, s]
    return exp


# ---------------------------------------------------------------------------------------------------------------------
# 6. the generic training path at the model level
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "tf32", "fp16"])
def test_2048_features_past_the_weight_gradient_grid_limit(prec):
    """2 048 scalar features and n = 8 001 rows: 32 weight-gradient splits, so the encoders' WGRAD group has 65 536 grid
    slices -- one over the limit.  Width-8 encoders are not tc-eligible, so every precision runs the simt launch, in two
    pieces; 'fp16' is off the fused envelope and takes the tf32 fallback."""
    cfg = O.DIBConfig([1] * 2048, [8], [16], 1, use_positional_encoding=False, feature_embedding_dimension=2)
    n = 7937 + 64
    rng = np.random.default_rng(20)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    x = rng.standard_normal((n, 2048)).astype(np.float32)
    y = rng.integers(0, 2, size=(n, 1)).astype(np.float32)
    eps = rng.standard_normal((n, 2048, 2)).astype(np.float32)
    m = build_model(cfg, precision=prec)
    if prec == "fp16":
        assert "encoders=grouped-wgmma-tf32" in m.kernel_info(n)
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    g, st = m.compute_gradients(x, y, eps=eps)
    g = g.cpu().numpy()
    g_ref, fr = O.train_grads(cfg, p, x, y, eps, 0.01, O.LOSS_BCE_LOGITS)
    tol, tol_var = (5e-5, 2e-4) if prec == "fp32" else (5e-3, 0.1)        # test_gpu_parity / test_gpu_tf32
    assert rel_err(g, g_ref) < tol
    pv = per_variable_errors(cfg, g, g_ref)
    assert pv.max() < tol_var, (int(pv.argmax()), float(pv.max()))
    np.testing.assert_allclose(st.cpu().numpy()[:2048] / n, fr.kl_per_feature, rtol=2e-5 if prec == "fp32" else 5e-3)


def _batch_split(n):
    """dib_api.cu batch_split: rows per weight-gradient split and the split count."""
    rps = max(math.ceil(n / 32), 256)
    rps = _ru(rps, 64)
    return rps, math.ceil(n / rps)


# Row isolation against the float64 oracle: max per-variable |g - oracle| / max |oracle|.  Measured on an H100 80GB HBM3
# (700 W): fp32 2.3e-6 (C0) / 1.1e-6 (hetero); tf32 with tanh (hetero) 1.7e-3; tf32 with relu (C0) 3.0e-1 -- 62 rows and
# an unrounded oracle: a tf32 rounding next to 0 flips relu' and moves one row's whole contribution to a 128 x 128 kernel.
# The step on the chosen rows alone runs the same per-row arithmetic, so it is held to fp32 summation order instead:
# measured 6.1e-7 (fp32) and 4.6e-7 (tf32), the tf32 C0 case included.
ROWISO_TOL = {("c0", "fp32"): 1e-4, ("hetero", "fp32"): 1e-4, ("c0", "tf32"): 0.6, ("hetero", "tf32"): 1e-2}
ROWISO_SELF = 1e-5


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("shape", ["c0", "hetero"])
def test_row_isolation_generic_path(prec, shape):
    """MSE, a linear head, beta = 0 and y = the model's own forward-only prediction: every row's gradient 2 (z - t) is
    exactly zero, so is the step.  Then y moves on chosen rows only -- both sides of every weight-gradient split boundary,
    rows 127 / 128, the first and the last row -- and the step must be those rows' contribution alone.  'hetero' has
    [2, 1, 2, 1] features: its first encoder layer runs on simt, the later ones on tc, in one stack."""
    if shape == "c0":
        cfg = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    else:
        cfg = O.DIBConfig([2, 1, 2, 1], [128, 128], [256, 256], 1, activation_fn="tanh")
    n = 20557
    rps, nsplit = _batch_split(n)
    assert nsplit == 30
    rng = np.random.default_rng(7)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)
    D = sum(cfg.feature_dimensionalities)
    x = rng.standard_normal((n, D)).astype(np.float32)
    eps = rng.standard_normal((n, cfg.number_features, 32)).astype(np.float32)
    m = build_model(cfg, precision=prec, loss="mse")
    m.set_flat_weights(p)
    m.beta.assign(0.0)
    y = np.asarray(m(x, eps=eps), dtype=np.float32)
    g0, st0 = m.compute_gradients(x, y, eps=eps)
    F = cfg.number_features
    assert float(st0[F]) == 0.0, ("training and forward-only predictions differ", float(st0[F]))
    assert int(torch.count_nonzero(g0)) == 0, int(torch.count_nonzero(g0))
    rows = {0, n - 1, 127, 128}
    for s in range(1, nsplit):
        rows |= {s * rps - 1, s * rps}
    rows = np.array(sorted(rows))
    y1 = y.copy()
    y1[rows] += np.where(np.arange(len(rows)) % 2 == 0, 0.25, -0.375).astype(np.float32)[:, None]
    g, st = m.compute_gradients(x, y1, eps=eps)
    g = g.cpu().numpy()
    want_loss = float(np.sum((y[rows].astype(np.float64) - y1[rows]) ** 2))
    assert abs(float(st[F]) - want_loss) <= 1e-6 * want_loss, (float(st[F]), want_loss)
    g_ref, _ = O.train_grads(cfg, p, x[rows], y1[rows], eps[rows], 0.0, O.LOSS_MSE, batch_for_mean=n)
    pv = per_variable_errors(cfg, g, g_ref)
    # the same rows as a batch of their own (one weight-gradient split), scaled by the same 1 / n
    m2 = build_model(cfg, precision=prec, loss="mse")
    m2.set_flat_weights(p)
    m2.beta.assign(0.0)
    g_alone, _ = m2.compute_gradients(x[rows], y1[rows], eps=eps[rows], global_batch=n)
    pv_self = per_variable_errors(cfg, g, g_alone.cpu().numpy())
    print(f"row isolation {shape} {prec}: {len(rows)} rows, worst per-variable error vs the oracle {pv.max():.3e} "
          f"(var {int(pv.argmax())}), vs the rows alone {pv_self.max():.3e} (var {int(pv_self.argmax())})")
    assert pv_self.max() < ROWISO_SELF, (int(pv_self.argmax()), float(pv_self.max()))
    assert pv.max() < ROWISO_TOL[(shape, prec)], (int(pv.argmax()), float(pv.max()))


@pytest.mark.parametrize("prec", ["fp32", "tf32", "fp16"])
def test_one_handle_through_changing_split_counts(prec):
    """One handle steps at n = 8 192 (32 splits), 300 (2) and 8 269 (26 splits of 320 rows); each step must equal a fresh
    handle's bit for bit, so no partial of a larger step leaks into a later reduction."""
    cfg = O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)
    rng = np.random.default_rng(8)
    p = O.glorot_uniform_params(cfg, rng)
    ns = (8192, 300, 8192 + 77)
    assert [_batch_split(n)[1] for n in ns] == [32, 2, 26]
    data = []
    for n in ns:
        x = rng.standard_normal((n, 16)).astype(np.float32)
        data.append((x, (x[:, :1] * x[:, 1:2] > 0).astype(np.float32)))
    m = build_model(cfg, precision=prec)
    m.kernel_info(max(ns))                              # size the handle for the largest step: no re-creation below
    m.set_flat_weights(p)
    m.beta.assign(0.01)
    handle = m._handle.value
    for (x, y) in data:
        g, st = m.compute_gradients(x, y, step=3)
        assert m._handle.value == handle
        f = build_model(cfg, precision=prec)
        f.set_flat_weights(p)
        f.beta.assign(0.01)
        gf, stf = f.compute_gradients(x, y, step=3)
        assert torch.equal(g, gf) and torch.equal(st, stf), (prec, x.shape[0])
        assert torch.isfinite(g).all()


def teardown_module(module):
    if _WORST:
        print("worst inexact FWD epilogue errors (fp32 ulps; tf32 ulps under round_out):",
              {f"{a}{' round_out' if r else ''}": round(v, 3) for (a, r), v in sorted(_WORST.items())})
