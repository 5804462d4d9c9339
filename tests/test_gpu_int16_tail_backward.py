"""GPU (H100): the dgrad stages of the fused integration tail (dib_int16_fwd2_kernel run in training with the layer-j1
dgrad and, when the embedding lies below, the embedding dgrad) against the same kernel without them followed by the
separate dib_int16_dgrad launches (debug_force_unfused(16)).  Every MMA keeps its operands and k order and every sum its
order, so predictions, gradients and statistics must be bit-identical."""
import numpy as np
import pytest
import torch

from oracle import dib_oracle as O
from tests.test_gpu_parity import build_model

pytestmark = pytest.mark.gpu


# F = 16 features -> a 512-wide embedding (C0), F = 12 -> 384 (C2: the last 128-column chunk of the embedding dgrad);
# integ [256] * 3: the layer below the fused pair is hidden, so the kernel runs only the layer-j1 dgrad
@pytest.mark.parametrize("precision,act,loss_name,F,integ", [
    ("fp16", "relu", "bce_logits", 16, [256, 256]),
    ("bf16", "relu", "bce_logits", 16, [256, 256]),
    ("fp16", "tanh", "mse", 12, [256, 256]),
    ("bf16", "tanh", "mse", 12, [256, 256]),
    ("fp16", "leaky_relu", "bce_logits", 16, [256, 256]),
    ("fp16", "tanh", "bce_logits", 16, [256, 256, 256]),
    ("bf16", "relu", "mse", 12, [256, 256, 256]),
])
def test_fused_tail_backward_is_bit_identical_to_separate_dgrads(precision, act, loss_name, F, integ):
    cfg = O.DIBConfig([1] * F, [128, 128], integ, 1, activation_fn=act)
    rng = np.random.default_rng(21)
    p = O.glorot_uniform_params(cfg, rng)
    p = p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)      # non-zero biases
    # a ragged last tile in fewer tiles than SMs; a ragged tile count that is not a multiple of the SM count
    for B in (128 * 3 + 17, 128 * 161 + 77):
        x = rng.standard_normal((B, F)).astype(np.float32)
        y = (x[:, :1] * x[:, 1:2] > 0).astype(np.float32) if loss_name == "bce_logits" else rng.standard_normal((B, 1)).astype(np.float32)
        res = {}
        for mask in (16, 0):
            m = build_model(cfg, precision=precision, loss=loss_name)
            m.debug_force_unfused(mask)
            want = "integration_tail=fwd2-head-dgrad" if mask == 0 else "integration_tail=fwd2-head"
            assert want in m.kernel_info(B), m.kernel_info(B)
            m.set_flat_weights(p)
            m.beta.assign(0.02)
            pred = m(x, step=3)                                         # forward only: the same kernel, no dgrad stages
            g, st = m.compute_gradients(x, y, step=3)
            assert torch.isfinite(g).all()
            res[mask] = (torch.as_tensor(np.asarray(pred)), g.clone(), st.clone())
        for a, b, what in zip(res[0], res[16], ("predictions", "gradients", "statistics")):
            assert torch.equal(a, b), (what, B)
