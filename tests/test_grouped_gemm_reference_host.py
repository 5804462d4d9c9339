"""CPU: the grouped GEMM's float64 reference (tests/grouped_gemm_reference.py) and fp_exact.round_tf32, its restatement of
cvt.rna.tf32.f32 -- and the exactness its operand generators claim -- and dib_create's refusal of more features than the
reparametrisation grid can index."""
import ctypes

import numpy as np
import pytest

from tests.fp_exact import act_grad32, dyadic, round_tf32
from tests.grouped_gemm_reference import act_source, ref_dgrad, ref_fwd, ref_wgrad


def _bits(u):
    return np.array(u, dtype=np.uint32).view(np.float32)


def _round_tf32_arith(x):
    """The same rounding by arithmetic: q = |x| / ulp_tf32(x), floor(q + 1/2) (ties away from zero), in float64."""
    x = np.asarray(x, np.float64)
    out = np.zeros_like(x)
    nz = x != 0
    e = np.floor(np.log2(np.abs(x[nz])))
    e = np.maximum(e, -126)                                  # subnormals share the smallest normal exponent's spacing
    ulp = np.exp2(e - 10)
    out[nz] = np.sign(x[nz]) * np.floor(np.abs(x[nz]) / ulp + 0.5) * ulp
    return out


@pytest.mark.parametrize("pattern,want", [
    (0x3F800000, 0x3F800000),   # 1.0: on the grid
    (0x3F800FFF, 0x3F800000),   # just below half of the dropped unit: down
    (0x3F801000, 0x3F802000),   # an exact tie with an even kept part: away from zero (not to even)
    (0x3F803000, 0x3F804000),   # an exact tie with an odd kept part: away from zero
    (0x3F801001, 0x3F802000),   # just above half: up
    (0xBF801000, 0xBF802000),   # a negative tie: away from zero, to the larger magnitude
    (0xBF800FFF, 0xBF800000),   # negative, below half: toward zero
    (0x3FFFF000, 0x40000000),   # 1.99993896: the carry runs into the exponent -> 2.0
    (0xBFFFF000, 0xC0000000),   # and negative -> -2.0
    (0x7F7FE000, 0x7F7FE000),   # the largest tf32 value stays
    (0x00001000, 0x00002000),   # a subnormal tie
    (0x80000000, 0x80000000),   # -0.0 keeps its sign
])
def test_round_tf32_hand_picked(pattern, want):
    got = round_tf32(_bits([pattern])).view(np.uint32)[0]
    assert got == want, (hex(pattern), hex(int(got)), hex(want))
    assert _round_tf32_arith(_bits([pattern]).astype(np.float64))[0] == _bits([want])[0]


def test_round_tf32_matches_arithmetic_rounding_and_passes_nan_inf():
    rng = np.random.default_rng(0)
    u = rng.integers(0, 0x7F7FE000, size=200000, dtype=np.uint32) | (rng.integers(0, 2, 200000, dtype=np.uint32) << 31)
    x = u.view(np.float32)
    got = round_tf32(x).astype(np.float64)
    np.testing.assert_array_equal(got, _round_tf32_arith(x.astype(np.float64)))
    assert np.all((round_tf32(x).view(np.uint32) & 0x1FFF) == 0)
    special = np.array([np.inf, -np.inf, np.nan], np.float32)
    assert np.array_equal(round_tf32(special)[:2], special[:2]) and np.isnan(round_tf32(special)[2])


def _f32_sum(v, order):
    """float32 running sum in the given order (every addition rounds to fp32)."""
    acc = np.float32(0)
    for t in v[order]:
        acc = np.float32(acc + t)
    return acc


def test_operands_are_exact_in_any_summation_order():
    """512-term dot products of dyadic operands (and the bias) summed in fp32 in shuffled orders equal the float64 sum,
    and o * act'(x) for every activation source is exact in one fp32 product."""
    rng = np.random.default_rng(1)
    for trial in range(40):
        T = 512
        a, w = dyadic(rng, T, dtype=np.float32), dyadic(rng, T, dtype=np.float32)
        if trial % 4 == 0:
            a, w = np.full(T, 1.0, np.float32), np.full(T, 1.0 if trial % 8 else -1.0, np.float32)     # |sum| at its bound
        prods = (a * w).astype(np.float32)
        assert np.array_equal(prods.astype(np.float64), a.astype(np.float64) * w.astype(np.float64))
        want = float(np.dot(a.astype(np.float64), w.astype(np.float64)))
        for _ in range(5):
            assert float(_f32_sum(prods, rng.permutation(T))) == want
        o = np.float32(want)
        x = (np.arange(-15, 16) / 16).astype(np.float32)           # every value act_source draws
        assert set(np.unique(act_source(rng, 4000))) == set(x)
        for act in ("relu", "tanh", "sigmoid", "elu", "leaky_relu"):
            g = act_grad32(act, x, 0.25)
            assert np.array_equal((o * g).astype(np.float64), float(o) * g.astype(np.float64)), act


def test_reference_rounds_only_where_the_kernels_round():
    rng = np.random.default_rng(2)
    a, w, b = dyadic(rng, (9, 33), dtype=np.float32), dyadic(rng, (33, 7), dtype=np.float32), dyadic(rng, 7, dtype=np.float32)
    z = a.astype(np.float64) @ w + b
    assert np.array_equal(ref_fwd(a, w, b, "linear", 0.2, 0), z.astype(np.float32))
    np.testing.assert_array_equal(ref_fwd(a, w, b, "leaky_relu", 0.2, 0),
                                  np.where(z > 0, z, np.float32(0.2) * z.astype(np.float32)).astype(np.float32))
    assert np.array_equal(ref_fwd(a, w, b, "relu", 0.2, 1), round_tf32(np.maximum(z, 0).astype(np.float32)))
    x = act_source(rng, (9, 33))
    dz = dyadic(rng, (9, 7), dtype=np.float32)
    want = (dz.astype(np.float64) @ w.T.astype(np.float64)) * (1 - x.astype(np.float64) ** 2)
    assert np.array_equal(ref_dgrad(dz, w, x, "tanh", 0.2, 0), want.astype(np.float32))
    h, d = dyadic(rng, (300, 5), dtype=np.float32), dyadic(rng, (300, 6), dtype=np.float32)
    dw, db = ref_wgrad(h, d, 300, 3, 128)
    assert np.array_equal(dw.sum(0).astype(np.float64), h.astype(np.float64).T @ d)
    assert np.array_equal(db[1], d[128:256].sum(0)) and np.array_equal(db[2], d[256:].sum(0))
    dw, db = ref_wgrad(h, d, 300, 4, 128)                     # a split past the batch: zero partials
    assert not dw[3].any() and not db[3].any()
    with pytest.raises(AssertionError, match="grid"):
        ref_fwd(a + np.float32(1 / 64), w, b, "linear", 0.2, 0)


def test_create_refuses_more_features_than_the_grid_can_index():
    """dib_create refuses number_features > 65 535 before it touches the device."""
    from dib_b200 import _lib
    lib = ctypes.CDLL(_lib.library_path())
    lib.dib_create.argtypes = _lib.SIGNATURES["dib_create"][1]
    lib.dib_last_error.restype = ctypes.c_char_p
    for F in (65536, 70000):
        fd = (ctypes.c_int32 * F)(*([1] * F))
        arch = (ctypes.c_int32 * 1)(4)
        cfg = _lib.DibConfig(abi_version=_lib.ABI_VERSION, number_features=F, feature_dimensionalities=fd,
                             number_encoder_layers=1, feature_encoder_architecture=arch, number_integration_layers=1,
                             integration_network_architecture=arch, output_dimensionality=1, use_positional_encoding=0,
                             number_positional_encoding_frequencies=1, feature_embedding_dimension=1, max_batch=1)
        h = ctypes.c_void_p()
        assert lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
        assert b"number_features" in lib.dib_last_error() and b"65535" in lib.dib_last_error()
        assert not h.value
