"""CPU checks of the float64 InfoNCE kernel reference (tests/infonce_stream_reference.py): it agrees with the oracles and with
autograd, its bounds vanish where the kernels' arithmetic is exact, and its bounds are tight enough that a kernel which
dropped a 32-column tile, the diagonal's -2/n or one column of a log-sum-exp would leave them."""
import math

import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests import infonce_oracle as IO
from tests import infonce_stream_reference as R


def _autograd(e1, e2, kind, T):
    a = torch.tensor(e1, dtype=torch.float64, requires_grad=True)
    b = torch.tensor(e2, dtype=torch.float64, requires_grad=True)
    loss = IO.torch_infonce(a, b, kind, T)
    loss.backward()
    return loss.item(), a.grad.numpy(), b.grad.numpy()


@pytest.mark.parametrize("kind", R.KINDS)
def test_agrees_with_the_oracles_away_from_ties(kind):
    e1, e2, _ = R.case_data(kind, 37, 5, "normal", seed=1)
    T = 0.5
    ref = R.reference(e1, e2, kind, T)
    n = e1.shape[0]
    for loss, d1, d2 in (O.infonce_loss_and_grads(e1, e2, kind, T)[:3], IO.infonce_loss_and_grads(e1, e2, kind, T, chunk=8)):
        assert abs(ref["loss"] / n - loss) < 1e-12
        np.testing.assert_allclose(ref["d1"], d1, rtol=0, atol=1e-12)
        np.testing.assert_allclose(ref["d2"], d2, rtol=0, atol=1e-12)


@pytest.mark.parametrize("regime", ["normal", "dyadic", "duplicate"])
@pytest.mark.parametrize("kind", R.KINDS)
def test_agrees_with_autograd_including_ties(kind, regime):
    """Dyadic operands tie everywhere under linf: the gradient is split between tied coordinates as torch.amax (and TF's
    reduce_max) split it.  The numpy oracles follow the same rule."""
    if kind == "l2" and regime == "duplicate":
        pytest.skip("the reference's expanded |a|^2 + |b|^2 - 2ab differs from the difference form at distance 0")
    e1, e2, T = R.case_data(kind, 12, 4, regime, seed=2)
    ref = R.reference(e1, e2, kind, T)
    loss, d1, d2 = _autograd(e1, e2, kind, T)
    scale = max(1.0, np.abs(d1).max(), np.abs(d2).max())
    assert abs(ref["loss"] / 12 - loss) < 1e-10 * max(1.0, abs(loss))
    np.testing.assert_allclose(ref["d1"], d1, rtol=0, atol=1e-10 * scale)
    np.testing.assert_allclose(ref["d2"], d2, rtol=0, atol=1e-10 * scale)
    for oracle in (O.infonce_loss_and_grads(e1, e2, kind, T)[:3], IO.infonce_loss_and_grads(e1, e2, kind, T, chunk=5)):
        if kind in ("l2", "l2sq") and regime == "duplicate":
            continue
        np.testing.assert_allclose(oracle[1], d1, rtol=0, atol=1e-10 * scale)
        np.testing.assert_allclose(oracle[2], d2, rtol=0, atol=1e-10 * scale)


def test_linf_ties_are_split_evenly():
    a = np.array([[1.0, -2.0, 2.0]], np.float32)
    b = np.array([[0.0, 0.0, 0.0]], np.float32)
    np.testing.assert_array_equal(R.linf_tie_weights32(a, b)[0, 0], [0.0, 0.5, 0.5])
    np.testing.assert_array_equal(O.linf_tie_weights(a[:, None, :] - b[None, :, :])[0, 0], [0.0, 0.5, 0.5])
    np.testing.assert_array_equal(R.linf_tie_weights32(b, b)[0, 0], [1 / 3] * 3)


@pytest.mark.parametrize("kind", ["l2sq", "l1", "linf"])
@pytest.mark.parametrize("T", [1.0, 2.0 ** -8, 2.0 ** 8])
def test_sigma_vanishes_on_exact_dyadic_operands(kind, T):
    e1, e2, _ = R.case_data(kind, 40, 33, "dyadic", seed=3)
    P = R.Pairs(e1, e2, kind, T)
    assert np.all(P.sigma == 0.0)
    lse = R.log_sum_exps(e1, e2, kind, T)
    assert np.all(lse["sigma_diag"] == 0.0)
    P3 = R.Pairs(e1, e2, kind, 0.3)                                          # 1/0.3 is not an fp32 value
    assert np.all(P3.sigma[P3.s != 0] > 0)


def test_sigma_is_positive_where_the_arithmetic_rounds():
    e1, e2, _ = R.case_data("l2sq", 20, 7, "normal", seed=4)
    for kind in R.KINDS:
        assert np.all(R.Pairs(e1, e2, kind, 1.0).sigma > 0), kind


@pytest.mark.parametrize("n,d", [s for s in R.GRAD_SHAPES if s[0] > 1])
@pytest.mark.parametrize("kind", R.KINDS)
def test_gradient_bounds_catch_a_dropped_tile_or_diagonal(kind, n, d):
    """At every gradient shape of the kernel test: leaving out any one 32-column tile, or the diagonal's -2/n, moves at least
    one element of d e1 and of d e2 out of its bound.  (At n = 1 the gradient is exactly 0 and is checked exactly.)"""
    if kind == "cosine" and d == 1:
        pytest.skip("cos = +-1 at d = 1: the exact gradient and every contribution to it are 0 (checked exactly on the GPU)")
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=5)
    lse = R.log_sum_exps(e1, e2, kind, T)
    args = [(e1, e2, lse["r"], lse["c"], lse["rho_r"], lse["rho_c"]), (e2, e1, lse["c"], lse["r"], lse["rho_c"], lse["rho_r"])]
    for side, (own, other, lo, lc, ro, rc) in enumerate(args):
        g, b, tiles, diag = R.side_gradient(own, other, kind, T, lo, lc, ro, rc, parts=True)
        assert np.any(np.abs(diag) > b), (kind, n, d, side, "diagonal")
        for t in range(tiles.shape[0]):
            assert np.any(np.abs(tiles[t]) > b), (kind, n, d, side, t)


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 63, 65, 100, 1000, 4097])
@pytest.mark.parametrize("kind", R.KINDS)
def test_log_sum_exp_bounds_catch_a_dropped_column(kind, n):
    d = 3 if n > 1000 else 17
    e1, e2, T = R.case_data(kind, n, d, "normal", seed=6)
    lse = R.log_sum_exps(e1, e2, kind, T)
    j = n - 1                                          # a column of the last, ragged tile
    P = R.Pairs(e1, e2, kind, T)
    s = np.delete(P.s, j, axis=1)
    with np.errstate(divide="ignore"):
        r_mut = np.log(np.exp(s - P.s.max(1, keepdims=True)).sum(1)) + P.s.max(1)
    assert np.any(np.abs(r_mut - lse["r"]) > lse["rho_r"]), (kind, n)
    np.testing.assert_allclose(lse["r"], np.log(np.exp(P.s).sum(1)), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(lse["c"], np.log(np.exp(P.s).sum(0)), rtol=1e-13, atol=1e-13)
    assert lse["rho_r"].max() < 1e-3 and math.isfinite(lse["rho_c"].max())
