"""CPU checks of the InfoNCE training path: the float64 oracle's joint gradient (model + output encoder) against autograd
and finite differences, the full-batch plan of fit, and the joint parameter layout (train.py:198)."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import dib_oracle as O
from tests import infonce_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _models_module():
    """dib_b200.models without loading the CUDA library: the batch-plan helpers are pure functions."""
    import dib_b200                                                        # noqa: F401  (the package; no device call)
    from dib_b200 import models
    return models


CFG = O.DIBConfig([2, 1], [16, 16], [24], 5, number_positional_encoding_frequencies=3, activation_fn="tanh",
                  feature_embedding_dimension=4)
YD, YARCH = 3, [12, 10]


def _case(seed, n=7):
    rng = np.random.default_rng(seed)
    p = IO.glorot(IO.infonce_param_shapes(CFG, YD, YARCH), rng)
    x = rng.standard_normal((n, 3))
    y = rng.standard_normal((n, YD))
    eps = rng.standard_normal((n, 2, 4))
    return p, x, y, eps


@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_oracle_infonce_grads_match_autograd_and_finite_differences(similarity):
    T = 0.1 if similarity == "cosine" else 1.0
    p, x, y, eps = _case(3)
    kw = dict(y_dimensionality=YD, y_encoder_architecture=YARCH, similarity=similarity, temperature=T)
    g, loss, kl = IO.infonce_train_grads(CFG, p, x, y, eps, 0.3, **kw)
    g_t, loss_t = IO.twin_infonce_grads(CFG, p, x, y, eps, 0.3, **kw)
    assert abs(loss - loss_t) < 1e-10
    np.testing.assert_allclose(g, g_t, rtol=1e-8, atol=1e-10)
    n_model = CFG.param_count()
    assert np.abs(g[n_model:]).max() > 0 and np.abs(g[:n_model]).max() > 0      # both networks receive a gradient

    def total(q):
        px, layers = IO.split_params(CFG, q, YD, YARCH)
        fr = O.forward(CFG, px, x, eps, 0.3)
        e2 = IO.output_encoder_forward(CFG, layers, y)
        return O.infonce_loss_and_grads(fr.pred, e2, similarity, T)[0] + 0.3 * fr.kl_per_feature.sum()

    rng = np.random.default_rng(1)
    idx = np.concatenate([rng.choice(n_model, 12, replace=False), n_model + rng.choice(p.size - n_model, 12, replace=False)])
    h = 1e-6
    for i in idx:
        e = np.zeros_like(p); e[i] = h
        fd = (total(p + e) - total(p - e)) / (2 * h)
        assert abs(fd - g[i]) < 1e-5 * max(1.0, abs(g[i])), (similarity, i, fd, g[i])


def test_epoch_batches_are_full_slices_of_the_permutation():
    m = _models_module()
    assert m.infonce_epoch_batches(10, 3) == [(0, 3), (3, 6), (6, 9)]
    assert m.infonce_epoch_batches(9, 3) == [(0, 3), (3, 6), (6, 9)]
    assert m.infonce_epoch_batches(4, 4) == [(0, 4)]
    with pytest.raises(ValueError):
        m.infonce_epoch_batches(3, 4)


@pytest.mark.parametrize("nv,b", [(10, 3), (9, 3), (2, 5), (5, 5), (1, 1)])
def test_validation_batches_wrap_around_the_repeated_permutation(nv, b):
    m = _models_module()
    plan = m.infonce_validation_batches(nv, b)
    assert plan.shape == (nv // b + 1, b)                                    # take(number_full_validation_batches + 1)
    flat = plan.ravel()
    np.testing.assert_array_equal(flat, np.arange(flat.size) % nv)          # the permutation, repeated end to end
    assert set(flat.tolist()) == set(range(nv)) or flat.size < nv


def test_joint_layout_is_model_then_output_encoder():
    shapes = IO.infonce_param_shapes(CFG, YD, YARCH)
    assert shapes[:len(CFG.param_shapes())] == CFG.param_shapes()
    w = YD * 3                                                               # PE with 2 sinusoid blocks
    assert shapes[len(CFG.param_shapes()):] == [(w, 12), (12,), (12, 10), (10,), (10, 5), (5,)]
    assert sum(int(np.prod(s)) for s in shapes) == CFG.param_count() + w * 12 + 12 + 12 * 10 + 10 + 10 * 5 + 5
    pend = O.DIBConfig([2, 1, 2, 1], [128, 128], [256, 256], 64)
    ps = IO.infonce_param_shapes(pend, 6, [128, 128])
    assert ps[len(pend.param_shapes())] == (30, 128) and ps[-1] == (64,)    # 6 -> PE 30 -> [128, 128] -> 64


def test_infonce_string_loss_points_to_the_loss_object():
    from dib_b200.keras_compat import InfoNCE, resolve_loss
    with pytest.raises(ValueError, match="losses.InfoNCE"):
        resolve_loss("infonce")
    assert resolve_loss(InfoNCE(6)) == "infonce"
    with pytest.raises(ValueError):
        InfoNCE(6, similarity="hamming")


@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_oracle_head_matches_autograd_on_integer_embeddings(similarity):
    """Integer-valued embeddings tie max_k |a_k - b_k| in many pairs: the 'linf' gradient is split evenly between the tied
    coordinates, as TF's reduce_max gradient and torch.amax split it."""
    import torch
    rng = np.random.default_rng(7)
    a, b = rng.integers(-3, 4, (6, 4)).astype(np.float64), rng.integers(-3, 4, (6, 4)).astype(np.float64)
    b[np.linalg.norm(b, axis=1) == 0, 0] = 1.0
    a[np.linalg.norm(a, axis=1) == 0, 0] = 1.0
    ta, tb = torch.tensor(a, requires_grad=True), torch.tensor(b, requires_grad=True)
    loss_t = IO.torch_infonce(ta, tb, similarity, 1.0)
    loss_t.backward()
    for loss, da, db in (O.infonce_loss_and_grads(a, b, similarity, 1.0)[:3], IO.infonce_loss_and_grads(a, b, similarity, 1.0, chunk=4)):
        assert abs(loss - loss_t.item()) < 1e-12
        if similarity in ("l2", "l2sq"):
            continue        # equal rows sit at the reference's clamp of |a|^2 + |b|^2 - 2ab, whose gradient the forms do not share
        np.testing.assert_allclose(da, ta.grad.numpy(), rtol=0, atol=1e-12)
        np.testing.assert_allclose(db, tb.grad.numpy(), rtol=0, atol=1e-12)
