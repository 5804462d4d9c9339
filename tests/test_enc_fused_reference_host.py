"""CPU: tests/enc_fused_reference.py -- the float64 restatement of the fused encoder kernels -- is the rounding oracle's
encoder (tests/fused16_oracle.py) tile by tile, its generators are exact, and every seeded kernel fault breaks a
comparison the GPU test makes."""
import numpy as np
import pytest

from oracle import dib_oracle as O
from tests import enc_fused_reference as R
from tests import fused16_oracle as Q
from tests.fp_exact import dyadic


def _case(fmt, fdims=(1, 2, 3), nfreq=1, act="relu", n=300, grid=5, seed=0, logvar_offset=-3.0, fault=None, density=1 / 16):
    """An exact-regime forward and backward through the reference.  Returns (ref results, inputs)."""
    rng = np.random.default_rng(seed)
    F = len(fdims)
    lay, count = R.layout(fdims, nfreq)
    enc = R.exact_params(rng, fdims, nfreq, logvar_offset, density)
    x = dyadic(rng, (n, sum(fdims)), 4, 2)
    x_off = np.concatenate([[0], np.cumsum(fdims)[:-1]]).astype(int)
    eps = dyadic(rng, (n, F, R.E), 4, 2)
    S, inv_batch, beta = 512.0, 1.0 / 512, 0.75
    d_emb = dyadic(rng, (n, F * R.E), 4, 4) / S
    img = R.pack(enc, fdims, nfreq, logvar_offset, fmt, fault if fault == "offset_after_round" else None)
    fw = R.forward(img, x, x_off, fdims, nfreq, act, 0.25, fmt, n, eps, grid, fault)
    g = (np.asarray(d_emb, np.float32) * np.float32(S)).astype(np.float64)
    parts = R.backward(img, fw["chains"], fdims, nfreq, act, 0.25, fmt, n, eps, g, beta, inv_batch, S, grid, lay, fault)
    return dict(fw=fw, parts=parts, img=img), dict(enc=enc, x=x, eps=eps, d_emb=d_emb, S=S, beta=beta, lay=lay, count=count,
                                                    fdims=fdims, nfreq=nfreq, act=act, n=n, grid=grid)


@pytest.mark.parametrize("act", ["relu", "linear", "leaky_relu"])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_reference_is_the_rounding_oracle(fmt, act):
    """Summed over slots, the per-(feature, slot) restatement equals fused16_oracle's encoder forward and backward, which
    equals dib_oracle without rounding (tests/test_fused16_oracle_host.py)."""
    fdims, nfreq = (1, 2, 3), 1
    ref, inp = _case(fmt, fdims, nfreq, act=act, grid=3, n=60 if act == "leaky_relu" else 300,
                     density=1 / 64 if act == "leaky_relu" else 1 / 16)
    cfg = O.DIBConfig(list(fdims), [128, 128], [256], 1, number_positional_encoding_frequencies=nfreq, activation_fn=act,
                      leaky_alpha=0.25, logvar_offset=-3.0)
    flat = np.concatenate([R.flatten_params(inp["enc"], inp["lay"], inp["count"]),
                           np.zeros(sum(int(np.prod(s)) for s in cfg.param_shapes()) - inp["count"])])
    fr = Q.forward(cfg, flat, inp["x"], inp["eps"], 0.0, fmt=fmt)
    assert np.array_equal(ref["fw"]["user_emb"], fr.emb)
    assert np.array_equal(ref["fw"]["emb16"], fr.cache["emb16"])
    np.testing.assert_allclose(ref["fw"]["kl_part"].sum(1) / inp["n"], fr.kl_per_feature, rtol=1e-15)
    g_emb = (np.asarray(inp["d_emb"], np.float32) * np.float32(inp["S"])).astype(np.float64)
    want = Q.encoder_backward(cfg, fr, inp["eps"], g_emb, inp["beta"], 1 / np.float32(1 / 512), inp["S"], fmt)
    got = np.zeros(inp["count"])
    for (f, s), blocks in ref["parts"].items():
        for b, v in blocks.items():
            got[int(inp["lay"][b][f]):int(inp["lay"][b][f]) + v.size] += v
    assert np.array_equal(got, want[:inp["count"]])


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_generators_are_exact(fmt):
    rng = np.random.default_rng(1)
    enc = R.exact_params(rng, (2,), 5, -3.0)
    img = R.pack(enc, (2,), 5, -3.0, fmt)
    W0p, W1, W2, Bb1, Bb2 = R.split_pack(img[0])
    assert np.array_equal(W1, enc[0]["W1"]) and np.array_equal(W2, enc[0]["W2"]) and np.array_equal(W0p[:10], enc[0]["W0"])
    assert np.all(Bb2[10, R.E:] == 0), "the packed logvar carrier must be 0 (lv = 0)"
    for e in R.pe_readout_params((3,), 5, "relu"):
        assert set(np.unique(e["W0"])) <= {-1.0, 0.0, 1.0}
    # the PE x picked for the exact regime: every sine farther than SIN_TOL from a midpoint, so r(sin) is the operand
    x = dyadic(rng, (4000, 2), 256, 64)
    ok = R.pe_exact(x, 2, 5, fmt)
    assert 0.5 < ok.mean() < 1.0


def test_schedule_covers_every_tile_once():
    for F, tiles in ((1, 7), (3, 5), (5, 3), (16, 2)):
        for grid in sorted({1, 2, max(F - 1, 1), F, F + 1, 2 * F - 1, F * tiles}):
            if grid > F * tiles:
                continue
            seen = {}
            for c, f, s, ts in R.schedule(F, grid, tiles):
                for t in ts:
                    assert (f, t) not in seen
                    seen[(f, t)] = s
            assert len(seen) == F * tiles
            assert [max(s for (ff, _), s in seen.items() if ff == f) + 1 for f in range(F)] == R.slots_per_feature(F, grid)


def _differs(a, b):
    return not np.array_equal(a, b)


def _parts_differ(pa, pb):
    return pa.keys() != pb.keys() or any(_differs(pa[k][b], pb[k][b]) for k in pa for b in pa[k])


# ---- every seeded fault breaks a comparison -----------------------------------------------------------------------------
@pytest.mark.parametrize("fault", ["wrong_slot", "slot_count"])
def test_fault_tile_credited_to_the_wrong_slot(fault):
    ref, _ = _case("fp16", n=700, grid=5)
    bad, _ = _case("fp16", n=700, grid=5, fault=fault)
    assert _differs(ref["fw"]["kl_part"], bad["fw"]["kl_part"]) and _parts_differ(ref["parts"], bad["parts"])


def test_fault_missed_restart_on_a_walking_ctas_second_feature():
    ref, _ = _case("fp16", fdims=(1, 2, 3, 1, 2), n=300, grid=2)
    bad, _ = _case("fp16", fdims=(1, 2, 3, 1, 2), n=300, grid=2, fault="no_restart")
    assert _parts_differ(ref["parts"], bad["parts"])


@pytest.mark.parametrize("fault", ["no_bias_carrier", "bias_after_act"])
def test_fault_bias_carrier(fault):
    ref, _ = _case("fp16", fault=None)
    bad, _ = _case("fp16", fault=fault)
    assert _differs(ref["fw"]["user_emb"], bad["fw"]["user_emb"])


def test_fault_relu_gate_from_the_unrounded_value():
    """A pre-activation below half the smallest fp16 subnormal rounds to 0: the gate of the rounded h is closed there, the
    gate of the fp32 value open."""
    fdims, nfreq, n = (1,), 1, 130
    enc = R.exact_params(np.random.default_rng(2), fdims, nfreq, 0.0)
    enc[0]["W0"][:] = 2.0 ** -14
    enc[0]["b0"][:] = 0.0
    x = np.full((n, 1), 2.0 ** -12)                                        # z1 = 2^-26: r() makes it 0
    eps = np.zeros((n, 1, R.E))
    img = R.pack(enc, fdims, nfreq, 0.0, "fp16")
    lay, _ = R.layout(fdims, nfreq)
    outs = []
    for fault in (None, "gate_unrounded"):
        fw = R.forward(img, x, [0], fdims, nfreq, "relu", 0.25, "fp16", n, eps, 1, fault)
        g = np.ones((n, R.E))
        outs.append(R.backward(img, fw["chains"], fdims, nfreq, "relu", 0.25, "fp16", n, eps, g, 0.0, 1.0, 1.0, 1, lay, fault))
    assert _parts_differ(*outs)


@pytest.mark.parametrize("fault", ["dl_without_half", "bs_without_S", "db0_unrouted"])
def test_fault_backward_epilogue(fault):
    ref, _ = _case("bf16", fault=None)
    bad, _ = _case("bf16", fault=fault)
    assert _parts_differ(ref["parts"], bad["parts"])


def test_fault_db2_written_by_both_warpgroups():
    ref, inp = _case("fp16", fault=None)
    bad, _ = _case("fp16", fault="db2_both")
    t = R.partial_table(ref["parts"], inp["lay"], inp["count"] + 64, 5, -7.0)
    tb = R.partial_table(bad["parts"], inp["lay"], inp["count"] + 64, 5, -7.0)
    assert _differs(t, tb)


def test_fault_ones_column_and_kl_past_the_batch_end():
    """The ones column on rows past n gives those rows a nonzero mu; the forward skips them, so the fault only shows where
    those rows are summed -- a KL sum over the whole last tile."""
    ref, _ = _case("fp16", n=300)
    bad, _ = _case("fp16", n=300, fault=("ones_past_n", "kl_past_n"))
    assert not _differs(ref["fw"]["kl_part"], _case("fp16", n=300, fault="kl_past_n")[0]["fw"]["kl_part"])
    assert _differs(ref["fw"]["kl_part"], bad["fw"]["kl_part"])


def test_fault_logvar_offset_after_rounding():
    ref, _ = _case("fp16", fault=None, logvar_offset=-2.9)
    bad_img = R.pack(R.exact_params(np.random.default_rng(0), (1, 2, 3), 1, -2.9), (1, 2, 3), 1, -2.9, "fp16",
                     "offset_after_round")
    assert _differs(ref["img"], bad_img)


def test_fault_pe_frequency_off_by_one_block():
    x = dyadic(np.random.default_rng(3), (64, 2), 64, 64)
    assert _differs(R.a0_operand(x, 64, 2, 5, "fp16"), R.a0_operand(x, 64, 2, 5, "fp16", "freq"))


@pytest.mark.parametrize("fault", ["swap_quad", "row_key"])
def test_fault_philox_noise(fault):
    good = R.philox_noise(7, 3, 2 ** 32 + 5, 40, 2)
    bad = R.philox_noise(7, 3, 2 ** 32 + 5, 40, 2, fault)
    assert (np.abs(good - bad) > R.Z_TOL * (1 + np.abs(good))).any()


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("d,nfreq", [(2, 5), (1, 15)])
def test_pe_layout_is_the_rounding_oracle(fmt, d, nfreq):
    """With a positional encoding, the reference's [pe | 1] column order and frequencies (pe_columns, sin_values) are
    dib_oracle.positional_encoding's: the backward's dW0 rows, which read every operand column, equal the oracle's.  The
    recipe of the GPU test: x whose sines lie away from a midpoint with |sin| >= 1/4, W0 = 0, integer gradients, beta 0."""
    rng = np.random.default_rng(7)
    n, F = 130, 1
    xs = dyadic(rng, (60 * n, d), 256, 128)
    s = R.sin_values(xs, d, nfreq)
    sine = np.array([fr != 0 for _, fr in R.pe_columns(d, nfreq)], bool)
    x = xs[R.pe_exact(xs, d, nfreq, fmt) & (np.abs(s[:, sine]) >= 0.25).all(1)][:n]
    lay, count = R.layout((d,), nfreq)
    enc = R.exact_params(rng, (d,), nfreq, -3.0, 1 / 32)
    enc[0]["W0"][:] = 0.0
    eps = dyadic(rng, (n, F, R.E), 2, 1)
    S = 256.0
    g = 2 * dyadic(rng, (n, R.E), 1, 1)
    img = R.pack(enc, (d,), nfreq, -3.0, fmt)
    fw = R.forward(img, x, [0], (d,), nfreq, "relu", 0.25, fmt, n, eps, 1)
    parts = R.backward(img, fw["chains"], (d,), nfreq, "relu", 0.25, fmt, n, eps, g, 0.0, 1 / S, S, 1, lay)
    cfg = O.DIBConfig([d], [128, 128], [256], 1, number_positional_encoding_frequencies=nfreq, logvar_offset=-3.0)
    flat = np.concatenate([R.flatten_params(enc, lay, count),
                           np.zeros(sum(int(np.prod(p)) for p in cfg.param_shapes()) - count)])
    fr = Q.forward(cfg, flat, x, eps, 0.0, fmt=fmt)
    assert np.array_equal(fw["chains"][0]["a0"][:n, :d * nfreq], fr.cache["enc"][0][0])
    want = Q.encoder_backward(cfg, fr, eps, g, 0.0, n, S, fmt)
    got = np.zeros(count)
    for (f, _), blocks in parts.items():
        for b, v in blocks.items():
            got[int(lay[b][f]):int(lay[b][f]) + v.size] += v
    assert np.array_equal(got, want[:count])
    assert np.any(got[int(lay["w0"][0]) + d * R.HID:int(lay["w0"][0]) + d * nfreq * R.HID] != 0), "the sine rows of dW0 are live"
