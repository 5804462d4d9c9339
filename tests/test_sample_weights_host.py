"""Per-sample weights of the compiled loss without a GPU: the weighted oracles of tests/sample_weight_oracle.py (identities that
pin them, and all-ones weights against the unweighted oracles they extend), the Keras class_weight map rule and the argument
checks of fit / evaluate / train_on_batch."""
import importlib

import numpy as np
import pytest

from oracle import dib_oracle as O
from tests import fused16_oracle as Q
from tests import sample_weight_oracle as SW

M = importlib.import_module("dib_b200.models")


def _case(loss, out, n=23, seed=0, out_act=None):
    cfg = O.DIBConfig([1, 2, 1], [16, 8], [12], out, feature_embedding_dimension=4, activation_fn="tanh",
                      output_activation_fn=out_act)
    rng = np.random.default_rng(seed)
    p = O.glorot_uniform_params(cfg, rng).astype(np.float64) + 0.05 * rng.standard_normal(cfg.param_count())
    x = rng.standard_normal((n, 4))
    eps = rng.standard_normal((n, 3, 4))
    if loss == O.LOSS_SPARSE_CE_LOGITS:
        y = rng.integers(0, out, n).astype(np.float64)
    elif loss == O.LOSS_MSE:
        y = rng.standard_normal((n, out))
    else:
        y = rng.integers(0, 2, (n, out)).astype(np.float64)
    return cfg, p, x, y, eps, rng


LOSSES = [(O.LOSS_BCE_LOGITS, 1, None), (O.LOSS_BCE_PROBS, 1, "sigmoid"), (O.LOSS_SPARSE_CE_LOGITS, 3, None),
          (O.LOSS_MSE, 2, None)]


@pytest.mark.parametrize("loss,out,out_act", LOSSES)
def test_all_ones_weights_equal_unweighted_exactly(loss, out, out_act):
    cfg, p, x, y, eps, _ = _case(loss, out, out_act=out_act)
    g0, f0 = O.train_grads(cfg, p, x, y, eps, 0.3, loss)
    g1, f1 = SW.train_grads(cfg, p, x, y, eps, 0.3, loss, np.ones(len(x)))
    assert np.array_equal(g0, g1) and f0.loss == f1.loss and f0.task_loss == f1.task_loss and f0.acc_sum == f1.acc_sum


@pytest.mark.parametrize("loss,out,out_act", LOSSES)
def test_integer_weights_equal_repeated_rows(loss, out, out_act):
    """beta = 0: the weighted batch is the batch with row i repeated w_i times, scaled by n_repeated / n."""
    cfg, p, x, y, eps, rng = _case(loss, out, out_act=out_act)
    w = rng.integers(0, 4, len(x)).astype(np.float64)
    w[:3] = [0, 1, 3]
    rep = np.repeat(np.arange(len(x)), w.astype(int))
    g, fr = SW.train_grads(cfg, p, x, y, eps, 0.0, loss, w)
    g_rep, fr_rep = O.train_grads(cfg, p, x[rep], y[rep], eps[rep], 0.0, loss)
    scale = len(rep) / len(x)
    np.testing.assert_allclose(g, g_rep * scale, rtol=1e-12, atol=1e-12 * np.abs(g).max())
    np.testing.assert_allclose(fr.task_loss, fr_rep.task_loss * scale, rtol=1e-12)


@pytest.mark.parametrize("loss,out,out_act", LOSSES)
def test_zero_weights_remove_the_task_term_not_the_kl(loss, out, out_act):
    cfg, p, x, y, eps, _ = _case(loss, out, out_act=out_act)
    g, fr = SW.train_grads(cfg, p, x, y, eps, 0.7, loss, np.zeros(len(x)))
    emb_dim = cfg.number_features * cfg.feature_embedding_dimension
    g_kl, fr_kl = O.train_grads(cfg, p, x, y, eps, 0.7, loss, d_emb=np.zeros((len(x), emb_dim)))
    n_enc = sum(int(np.prod(s)) for s in cfg.param_shapes()[:2 * 3 * cfg.number_features])
    assert fr.task_loss == 0.0 and fr.loss == pytest.approx(O.ib_loss(cfg, 0.7, fr.kl_per_feature), rel=1e-15)
    assert not np.any(g[n_enc:])                                        # the integration network gets nothing
    np.testing.assert_allclose(g[:n_enc], g_kl[:n_enc], rtol=1e-12, atol=1e-15)
    assert np.any(g[:n_enc])                                            # the KL still trains the encoders
    # and one zero row: its task term is gone, the others are untouched
    w = np.ones(len(x)); w[5] = 0.0
    keep = np.arange(len(x)) != 5
    _, fr1 = SW.train_grads(cfg, p, x, y, eps, 0.0, loss, w)
    _, fr2 = O.train_grads(cfg, p, x[keep], y[keep], eps[keep], 0.0, loss)
    np.testing.assert_allclose(fr1.task_loss, fr2.task_loss * (len(x) - 1) / len(x), rtol=1e-12)


@pytest.mark.parametrize("loss,out,out_act", LOSSES)
def test_weighted_gradient_matches_finite_differences(loss, out, out_act):
    cfg, p, x, y, eps, rng = _case(loss, out, n=9, out_act=out_act)
    w = rng.uniform(0, 5, len(x))
    w[2] = 0.0
    g, _ = SW.train_grads(cfg, p, x, y, eps, 0.2, loss, w)
    f = lambda q: SW.forward(cfg, q, x, eps, 0.2, y, loss, w).loss
    for k in rng.choice(p.size, 25, replace=False):
        h = 1e-6
        e = np.zeros_like(p); e[k] = h
        fd = (f(p + e) - f(p - e)) / (2 * h)
        assert fd == pytest.approx(g[k], rel=1e-5, abs=1e-8), k


@pytest.mark.parametrize("fmt", [None, "fp16", "bf16"])
@pytest.mark.parametrize("loss,out,out_act", LOSSES)
def test_fused16_weighted_oracle_with_unit_weights_is_the_unweighted_one(loss, out, out_act, fmt):
    cfg = O.DIBConfig([1] * 3, [16, 16], [24, 24], out, feature_embedding_dimension=4, activation_fn="tanh",
                      output_activation_fn=out_act)
    _, p, x, y, _, rng = _case(loss, out, n=13, out_act=out_act)
    p = O.glorot_uniform_params(cfg, rng).astype(np.float64)
    x = x[:, :3]
    eps = rng.standard_normal((13, 3, 4))
    g0, f0 = Q.train_grads(cfg, p, x, y, eps, 0.3, loss, fmt=fmt)
    g1, f1 = SW.fused16_train_grads(cfg, p, x, y, eps, 0.3, loss, np.ones(13), fmt=fmt)
    assert np.array_equal(g0, g1) and np.array_equal(f0.cache["d_emb16"], f1.cache["d_emb16"])
    assert f0.task_loss == f1.task_loss and f0.cache["loss_sum"] == f1.cache["loss_sum"] and f0.acc_sum == f1.acc_sum
    # and with weights, without rounding it is the float64 weighted oracle
    w = rng.uniform(0, 4, 13)
    g2, _ = SW.fused16_train_grads(cfg, p, x, y, eps, 0.3, loss, w)
    g3, _ = SW.train_grads(cfg, p, x, y, eps, 0.3, loss, w)
    np.testing.assert_allclose(g2, g3, rtol=1e-10, atol=1e-12 * np.abs(g3).max())


@pytest.mark.parametrize("varlen", [False, True])
def test_set_transformer_weighted_oracle_with_unit_weights_is_the_unweighted_one(varlen):
    from tests import set_transformer_oracle as STO
    from tests import set_transformer_varlen_oracle as VO
    cfg = STO.STConfig(particle_feature_dimensions=2, particle_encoder_arch_spec=[8], bottleneck_dimension=4, number_particles=5,
                       key_dim=4, number_heads=2, number_attention_blocks=1, ff_arch_per_block=[6, 4], final_processing_arch=[6],
                       number_positional_encoding_frequencies=2)
    rng = np.random.default_rng(4)
    B = 7
    p = STO.init_params(cfg, rng).astype(np.float64)
    x = rng.standard_normal((B, 5, 2))
    eps = rng.standard_normal((B, 5, 4))
    y = (rng.random((B, 1)) > 0.5).astype(np.float64)
    sizes = rng.integers(1, 6, B).astype(np.int32) if varlen else None
    if varlen:
        g0, f0 = VO.train_grads(cfg, p, x, y, eps, sizes, 0.1)
    else:
        g0, f0 = STO.train_grads(cfg, p, x, y, eps, 0.1)
    g1, f1 = SW.set_transformer_train_grads(cfg, p, x, y, eps, 0.1, O.LOSS_BCE_LOGITS, np.ones(B), sizes=sizes)
    assert np.array_equal(g0, g1) and f0.task_loss == f1.task_loss and f0.loss == f1.loss
    # integer weights, beta = 0: the sets repeated w_i times, scaled by n_repeated / n
    w = rng.integers(0, 4, B).astype(np.float64)
    rep = np.repeat(np.arange(B), w.astype(int))
    g, _ = SW.set_transformer_train_grads(cfg, p, x, y, eps, 0.0, O.LOSS_BCE_LOGITS, w, sizes=sizes)
    g_rep, _ = (VO.train_grads(cfg, p, x[rep], y[rep], eps[rep], sizes[rep], 0.0) if varlen else
                STO.train_grads(cfg, p, x[rep], y[rep], eps[rep], 0.0))
    np.testing.assert_allclose(g, g_rep * len(rep) / B, rtol=1e-10, atol=1e-12 * np.abs(g).max())


def test_weighted_fit_history_is_the_weighted_loss():
    cfg, p, x, y, eps, rng = _case(O.LOSS_BCE_LOGITS, 1, n=20)
    w = rng.uniform(0, 3, len(x))
    eps_fn = lambda step, ids: np.random.default_rng(step).standard_normal((len(ids), 3, 4))
    _, h0 = O.fit(cfg, p, x, y, loss=O.LOSS_BCE_LOGITS, epochs=2, batch_size=8, lr=1e-3, eps_fn=eps_fn,
                  validation_data=(x[:6], y[:6]))
    _, h1 = SW.fit(cfg, p, x, y, loss=O.LOSS_BCE_LOGITS, epochs=2, batch_size=8, lr=1e-3, eps_fn=eps_fn,
                  validation_data=(x[:6], y[:6], np.ones(6)), sample_weight=np.ones(len(x)))
    assert h0 == h1                                                        # all-ones: exactly O.fit's unweighted run
    _, h3 = SW.fit(cfg, p, x, y, loss=O.LOSS_BCE_LOGITS, epochs=2, batch_size=8, lr=1e-3, eps_fn=eps_fn,
                   validation_data=(x[:6], y[:6]))
    assert h0 == h3
    _, h2 = SW.fit(cfg, p, x, y, loss=O.LOSS_BCE_LOGITS, epochs=1, batch_size=8, lr=1e-3, eps_fn=eps_fn, sample_weight=w)
    assert h2["loss"][0] != h0["loss"][0] and h2["accuracy"][0] == h0["accuracy"][0]   # accuracy stays unweighted


# ---------------------------------------------------------------------------------------------------------------------
# class_weight: Keras' _make_class_weight_map_fn, restated directly
# ---------------------------------------------------------------------------------------------------------------------
def _keras_map(class_weight, y, sw=None):
    class_ids = list(sorted(class_weight.keys()))
    if class_ids != list(range(len(class_ids))):
        raise ValueError("keys")
    table = np.asarray([class_weight[int(c)] for c in class_ids], dtype=np.float32)
    y = np.asarray(y)
    if y.ndim == 2 and y.shape[1] > 1:
        cls = np.argmax(y, axis=1)
    else:
        cls = np.reshape(y, (-1,)).astype(np.int64)               # tf.cast(float -> int64) truncates toward zero
    cw = table[cls]
    return cw if sw is None else np.asarray(sw, np.float32).reshape(-1) * cw


CW = {0: 1.0, 1: 20.0, 2: 0.5}


@pytest.mark.parametrize("y", [
    np.eye(3, dtype=np.float32)[[0, 2, 1, 1, 0]],                                 # one-hot: argmax
    np.array([[0.1, 0.7, 0.2], [0.5, 0.2, 0.3]], np.float32),                     # soft labels: argmax
    np.array([[0.], [2.], [1.], [1.]], np.float32),                               # [n, 1]
    np.array([0.0, 1.7, 2.2, 0.9, 2.999], np.float32),                            # float labels truncate
    np.array([0, 2, 1], np.int64),
])
def test_class_weight_rows_is_keras_map(y):
    np.testing.assert_array_equal(M.class_weight_rows(y, CW), _keras_map(CW, y))
    sw = np.linspace(0.0, 3.0, len(y)).astype(np.float32)
    np.testing.assert_array_equal(M.class_weight_rows(y, CW, sw), _keras_map(CW, y, sw))
    np.testing.assert_array_equal(M.class_weight_rows(y, CW, sw[:, None]), _keras_map(CW, y, sw))


@pytest.mark.parametrize("cw", [{1: 1.0, 2: 3.0}, {0: 1.0, 2: 3.0}, {0: 1.0, -1: 2.0}, {}, [1.0, 2.0], {0: -1.0},
                                {0: float("nan")}])
def test_class_weight_key_set_and_values_are_checked(cw):
    with pytest.raises(ValueError):
        M.check_class_weight(cw)


@pytest.mark.parametrize("y", [np.array([0., 3.]), np.array([-1., 0.]), np.array([np.nan, 0.]), np.array([[0.], [5.]]),
                               np.zeros((2, 1, 1))])
def test_class_labels_outside_the_table_raise(y):
    with pytest.raises(ValueError):
        M.class_weight_rows(y, CW)


@pytest.mark.parametrize("w,n", [(np.ones(4), 5), (np.ones((5, 2)), 5), (np.ones((1, 5)), 5), (-np.ones(5), 5),
                                 (np.array([1, 1, np.nan, 1, 1]), 5), (np.array([1, 1, np.inf, 1, 1]), 5),
                                 (np.array(["a"] * 5), 5)])
def test_sample_weight_shape_and_values_are_checked(w, n):
    with pytest.raises(ValueError):
        M.check_sample_weights(w, n)


def test_sample_weight_accepted_shapes():
    np.testing.assert_array_equal(M.check_sample_weights(np.arange(4), 4), np.arange(4, dtype=np.float32))
    np.testing.assert_array_equal(M.check_sample_weights(np.arange(4.)[:, None], 4), np.arange(4, dtype=np.float32))
    assert M.check_sample_weights(np.zeros(3, bool), 3).dtype == np.float32


@pytest.mark.parametrize("kind,out,cw", [("infonce", 4, False), ("external", 1, False), ("infonce", 4, True),
                                         ("mse", 1, True), ("bce_logits", 2, True), ("bce_probs", 3, True)])
def test_refused_losses(kind, out, cw):
    with pytest.raises(ValueError):
        M.check_weighted_loss(kind, out, class_weight=cw)


@pytest.mark.parametrize("kind,out,cw", [("bce_logits", 1, True), ("bce_probs", 1, True), ("sparse_ce_logits", 8, True),
                                         ("mse", 6, False), ("bce_logits", 3, False)])
def test_accepted_losses(kind, out, cw):
    M.check_weighted_loss(kind, out, class_weight=cw)
