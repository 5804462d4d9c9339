"""CPU checks of the float64 elementwise-kernel reference (tests/elementwise_reference.py): it agrees with the model oracle
(oracle/dib_oracle.py) and with torch autograd, its exactness claims hold, and its bounds are tight enough that a kernel with
one of the seeded faults below would leave them."""
import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from oracle import philox
from tests import elementwise_reference as R


def _ml(rng, F, n, E, s=1.0):
    mu = rng.normal(0, s, (F, n, E)).astype(np.float32)
    lv = rng.normal(0, s, (F, n, E)).astype(np.float32)
    return mu, lv


def _breaks(got, ref, bound):
    return bool((np.abs(np.asarray(got, np.float64) - ref) > bound).any())


# ---- agreement with the oracle and autograd ---------------------------------------------------------------------------------
def test_reparam_agrees_with_the_oracle_and_autograd():
    rng = np.random.default_rng(1)
    F, n, E = 3, 300, 5
    mu, lv = _ml(rng, F, n, E)
    z = rng.standard_normal((F, n, E)).astype(np.float32)
    du = rng.standard_normal((F, n, E))
    beta, ib = 0.3, 1.0 / n
    f = R.reparam_forward(mu, lv, z)
    m64, l64, z64 = (a.astype(np.float64) for a in (mu, lv, z))
    np.testing.assert_allclose(f["u"], m64 + np.exp(l64 / 2.0) * z64, rtol=0, atol=1e-12)
    kl_or = (0.5 * (mu.astype(np.float64) ** 2 + (np.expm1(lv.astype(np.float64)) - lv))).sum(-1).mean(-1)
    np.testing.assert_allclose(f["kl"].sum(-1).mean(-1), kl_or, rtol=1e-12)
    np.testing.assert_allclose(f["kl_part"].sum(-1) / n, kl_or, rtol=1e-12)
    tm, tl = torch.tensor(mu, dtype=torch.float64, requires_grad=True), torch.tensor(lv, dtype=torch.float64, requires_grad=True)
    u = tm + torch.exp(tl / 2) * torch.tensor(z, dtype=torch.float64)
    kl = (0.5 * (tm ** 2 + torch.exp(tl) - tl - 1)).sum()
    b32 = float(np.float32(beta)) * float(np.float32(ib))
    ((u * torch.tensor(du)).sum() + b32 * kl).backward()
    b = R.reparam_backward(mu, lv, z, du, beta, ib)
    np.testing.assert_allclose(b["dmu"], tm.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(b["dlv"], tl.grad.numpy(), rtol=0, atol=1e-12)


@pytest.mark.parametrize("kind", ["bce_logits", "sparse_ce_logits", "mse", "bce_probs"])
@pytest.mark.parametrize("C", [1, 3, 16])
def test_loss_agrees_with_the_oracle(kind, C):
    if kind == "sparse_ce_logits" and C == 1:
        C = 2
    rng = np.random.default_rng(2)
    n = 300
    z = rng.standard_normal((n, C))
    if kind == "bce_probs":
        z = 1 / (1 + np.exp(-z))
    y = rng.integers(0, C, n).astype(np.float64) if kind == "sparse_ce_logits" else (rng.random((n, C)) > 0.5).astype(np.float64)
    ok = O.LOSS_SPARSE_CE_LOGITS if kind == "sparse_ce_logits" else {"bce_logits": O.LOSS_BCE_LOGITS, "mse": O.LOSS_MSE,
                                                                      "bce_probs": O.LOSS_BCE_PROBS}[kind]
    r = R.loss(kind, "linear", 0.0, z, y, 1.0)
    np.testing.assert_allclose(r["row_loss"], O.task_loss_per_sample(ok, z, y), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["dz"], O.task_loss_grad(ok, z, y), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["acc_part"].sum(), O.accuracy_count(ok, z, y), rtol=1e-12)
    # autograd of the float64 loss
    tz = torch.tensor(z, requires_grad=True)
    if kind == "sparse_ce_logits":
        lt = torch.nn.functional.cross_entropy(tz, torch.tensor(y, dtype=torch.int64), reduction="sum")
    elif kind == "bce_logits":
        lt = torch.nn.functional.binary_cross_entropy_with_logits(tz, torch.tensor(y), reduction="none").mean(-1).sum()
    elif kind == "mse":
        lt = ((tz - torch.tensor(y)) ** 2).mean(-1).sum()
    else:
        e = R.KERAS_EPS
        pc = torch.clamp(tz, e, R.ONE_M_EPS)
        lt = (-(torch.tensor(y) * torch.log(pc + e) + (1 - torch.tensor(y)) * torch.log(1 - pc + e))).mean(-1).sum()
    lt.backward()
    np.testing.assert_allclose(r["row_loss"].sum(), float(lt), rtol=1e-12)
    np.testing.assert_allclose(r["dz"], tz.grad.numpy(), rtol=1e-12, atol=1e-14)


def test_sparse_labels_follow_one_rule():
    z = np.array([[1.0, 3.0, 3.0], [0.5, 0.0, 2.0], [2.0, 1.0, 0.0], [1.0, 2.0, 3.0], [0.0, 1.0, 0.0], [0.0, 1.0, 0.0],
                  [1.0, 0.0, 0.0]])
    y = np.array([1.0, 2.7, -0.5, 3.0, -1.0, np.nan, 0.0])
    r = R.loss("sparse_ce_logits", "linear", 0.0, z, y, 1.0)
    bad = np.array([False, False, False, True, True, True, False])
    assert np.array_equal(np.isnan(r["row_loss"]), bad)
    assert np.array_equal(np.isnan(r["dz"]).all(-1), bad) and not np.isnan(r["dz"][~bad]).any()
    assert r["row_acc"].tolist() == [1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]      # ties: first maximum; 2.7 never hits
    assert O.accuracy_count(O.LOSS_SPARSE_CE_LOGITS, z, y) == r["row_acc"].sum() == 2.0
    np.testing.assert_array_equal(np.isnan(O.task_loss_per_sample(O.LOSS_SPARSE_CE_LOGITS, z, y)), bad)
    np.testing.assert_array_equal(np.isnan(O.task_loss_grad(O.LOSS_SPARSE_CE_LOGITS, z, y)).all(-1), bad)
    assert R.sparse_label(y, 3).tolist() == [1, 2, 0, -1, -1, -1, 0]


# ---- exactness claims -------------------------------------------------------------------------------------------------------
def test_dropout_restatement_is_the_fp32_product():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((7, 9)).astype(np.float32)
    for rate in (0.0, 2.0 ** -24, 0.5, 0.3):
        keep = philox.dropout_keep(5, 2, np.arange(7), 1, 0, 9, np.float32(rate))
        got = R.dropout(x, keep, rate)
        if rate == 0.5:
            np.testing.assert_array_equal(got, np.where(keep, 2.0 * x, 0.0))
        if rate == 0.0:
            np.testing.assert_array_equal(got, x)
        assert np.array_equal(got == 0, ~keep | (x == 0)) or rate == 0.0


def test_accuracy_and_reductions_are_exact():
    rng = np.random.default_rng(4)
    z = rng.standard_normal((600, 4))
    y = (rng.random((600, 4)) > 0.5).astype(np.float64)
    r = R.loss("bce_logits", "linear", 0.0, z, y, 1.0 / 600)
    assert not r["acc_part_bound"].any() and not r["row_acc_bound"].any()
    r3 = R.loss("bce_logits", "linear", 0.0, z[:, :3], y[:, :3], 1.0 / 600)
    assert r3["row_acc_bound"].any()                          # 1/3 is not exact in fp32
    src = rng.integers(-1000, 1000, (65, 4097)).astype(np.float32)
    for order in (np.arange(65), np.arange(65)[::-1], rng.permutation(65)):
        acc = np.zeros(4097, np.float32)
        for k in order:
            acc += src[k]
        np.testing.assert_array_equal(acc, src.astype(np.float64).sum(0))


def test_the_kl_bound_holds_for_the_new_term_and_vanishes_only_at_zero():
    rng = np.random.default_rng(5)
    for s in (1e-4, 1e-3, 0.05, 1.0, 8.0):
        mu, lv = _ml(rng, 1, 4096, 1, s)
        f = R.reparam_forward(mu, lv, np.zeros_like(mu))
        got = R.kl_term_fp32(mu, lv)
        assert not _breaks(got, f["kl"], f["kl_bound"]), s
        assert (f["kl_bound"] > 0).all()


# ---- seeded faults ----------------------------------------------------------------------------------------------------------
def test_the_old_kl_formula_breaks_the_bound_at_small_scale():
    rng = np.random.default_rng(6)
    mu, lv = _ml(rng, 1, 4096, 1, 1e-4)
    f = R.reparam_forward(mu, lv, np.zeros_like(mu))
    assert _breaks(R.kl_term_old_fp32(mu, lv), f["kl"], f["kl_bound"])


def test_a_label_from_the_neighbouring_row_breaks_the_bound():
    rng = np.random.default_rng(7)
    z = rng.standard_normal((300, 5))
    y = rng.integers(0, 5, 300).astype(np.float64)
    r = R.loss("sparse_ce_logits", "linear", 0.0, z, y, 1.0 / 300)
    f = R.loss("sparse_ce_logits", "linear", 0.0, z, np.roll(y, -1), 1.0 / 300)
    assert _breaks(f["row_loss"], r["row_loss"], r["row_loss_bound"])
    assert _breaks(f["dz"], r["dz"], r["dz_bound"])


@pytest.mark.parametrize("act", ["tanh", "sigmoid", "elu"])
def test_a_missing_act_grad_or_one_over_out_breaks_the_bound(act):
    rng = np.random.default_rng(8)
    z = {"tanh": np.tanh(rng.standard_normal((300, 3))), "sigmoid": rng.random((300, 3)) * 0.9 + 0.05,
         "elu": rng.uniform(-0.9, 0.9, (300, 3))}[act]
    y = (rng.random((300, 3)) > 0.5).astype(np.float64)
    r = R.loss("mse", act, 0.0, z, y, 1.0 / 300)
    no_act = R.loss("mse", "linear", 0.0, z, y, 1.0 / 300)
    assert _breaks(no_act["dz"], r["dz"], r["dz_bound"])
    assert _breaks(r["dz"] * 3, r["dz"], r["dz_bound"])                       # without the 1/out factor
    assert _breaks(r["row_loss"] * 3, r["row_loss"], r["row_loss_bound"])


def test_a_dropped_last_row_of_a_block_breaks_the_bound():
    rng = np.random.default_rng(9)
    mu, lv = _ml(rng, 2, 512, 4)
    f = R.reparam_forward(mu, lv, rng.standard_normal(mu.shape))
    real = np.ones(512, bool)
    real[255] = False
    g = R.reparam_forward(mu, lv, rng.standard_normal(mu.shape), real=real)
    assert _breaks(g["kl_part"], f["kl_part"], f["kl_part_bound"])
    z = rng.standard_normal((512, 2))
    y = (rng.random((512, 2)) > 0.5).astype(np.float64)
    r = R.loss("bce_logits", "linear", 0.0, z, y, 1.0 / 512)
    assert _breaks(r["loss_part"] - np.array([r["row_loss"][255], 0.0]), r["loss_part"], r["loss_part_bound"])


def test_a_skipped_or_double_counted_row_changes_an_exact_reduction():
    rng = np.random.default_rng(10)
    src = rng.integers(-100, 100, (9, 33)).astype(np.float64)
    ref = src.sum(0)
    assert (src[:8].sum(0) != ref).any() and (src.sum(0) + src[8] != ref).any()


def test_dropout_with_the_wrong_layer_or_feature_changes_the_mask():
    x = np.ones((64, 13), np.float32)
    keep = philox.dropout_keep(7, 3, np.arange(64), 1, 2, 13, np.float32(0.5))
    ref = R.dropout(x, keep, 0.5)
    for f, layer in ((0, 2), (1, 1), (2, 2)):
        wrong = R.dropout(x, philox.dropout_keep(7, 3, np.arange(64), f, layer, 13, np.float32(0.5)), 0.5)
        assert (wrong != ref).any()


def test_a_pe_frequency_off_by_one_block_breaks_the_bound():
    rng = np.random.default_rng(11)
    x = rng.uniform(-3, 3, (300, 2)).astype(np.float32)
    src = np.array([0, 1, 0, 1, 0, 1])
    freq = np.array([0, 0, 2, 2, 4, 4])
    ref, b = R.pe(x, src, freq, 0, 6)
    bad, _ = R.pe(x, src, np.array([0, 0, 4, 4, 8, 8]), 0, 6)
    assert _breaks(bad, ref, b)


# ---- public entry points' references ----------------------------------------------------------------------------------------
def test_pairwise_gaussian_reference_agrees_with_the_direct_formulas():
    rng = np.random.default_rng(20)
    E = 3
    ml1 = np.concatenate([rng.standard_normal((5, E)), rng.uniform(-2, 2, (5, E))], 1)
    ml2 = np.concatenate([rng.standard_normal((7, E)), rng.uniform(-2, 2, (7, E))], 1)
    a, la, b, lb = ml1[:, None, :E], ml1[:, None, E:], ml2[None, :, :E], ml2[None, :, E:]
    sbar = 0.5 * (np.exp(la) + np.exp(lb))
    bh = (0.125 * ((a - b) ** 2 / sbar).sum(-1) + 0.5 * (np.log(sbar) - 0.5 * (la + lb)).sum(-1))
    kl = 0.5 * ((lb - la - 1) + np.exp(la - lb) + (b - a) ** 2 * np.exp(-lb)).sum(-1)
    np.testing.assert_allclose(R.pairwise_gaussian(0, ml1, ml2)["D"], bh, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(R.pairwise_gaussian(1, ml1, ml2)["D"], kl, rtol=1e-12, atol=1e-14)
    same = R.pairwise_gaussian(0, ml1, ml1)
    assert not np.diag(same["D"]).any() and (same["D_bound"] > 0).all()


def test_optimizer_references_agree_with_the_keras_formulas():
    rng = np.random.default_rng(21)
    w, g = rng.standard_normal(50), rng.standard_normal(50)
    b1, b2, eps, lr = (float(np.float32(x)) for x in (0.9, 0.999, 1e-7, 1e-3))
    m, v2 = (1 - b1) * g, (1 - b2) * g * g                      # tf.keras Adam, step 1 from zero moments
    r = R.adam(w, g, np.zeros(50), np.zeros(50), 1e-3, 1, 0.9, 0.999, 1e-7)
    np.testing.assert_allclose(r["w"], w - lr * np.sqrt(1 - b2) / (1 - b1) * m / (np.sqrt(v2) + eps), rtol=1e-14)
    v = rng.standard_normal(50)
    r = R.sgd(w, g, v, 0.01, 0.9, True)
    vv = float(np.float32(0.9)) * v - float(np.float32(0.01)) * g
    np.testing.assert_allclose(r["w"], w + float(np.float32(0.9)) * vv - float(np.float32(0.01)) * g, rtol=1e-14)
    ms, mom = rng.random(50), rng.standard_normal(50)
    r = R.rmsprop(w, g, ms, mom, 0.01, 0.9, 0.5, 1e-7)
    rho, lr = float(np.float32(0.9)), float(np.float32(0.01))
    ms1 = rho * ms + (1 - rho) * g * g
    np.testing.assert_allclose(r["w"], w - (0.5 * mom + lr * g / np.sqrt(ms1 + float(np.float32(1e-7)))), rtol=1e-14)
    assert (r["w_bound"] > 0).all()


def test_a_missing_adam_bias_correction_breaks_the_bound():
    rng = np.random.default_rng(22)
    w, g = rng.standard_normal(300), rng.standard_normal(300)
    r = R.adam(w, g, np.zeros(300), np.zeros(300), 1e-3, 1, 0.9, 0.999, 1e-7)
    wrong = w - 1e-3 * (0.1 * g) / (np.sqrt(0.001 * g * g) + 1e-7)
    assert _breaks(wrong, r["w"], r["w_bound"])
