"""TEST INFRASTRUCTURE ONLY -- the model builders, data cases and device helpers that several GPU suites share.  Not collected
by pytest (no test_ prefix).  Importing it neither loads the library nor touches a device: dib_b200 and torch are imported
inside the functions that need them, so host tests can import it on a machine without a GPU."""
import ctypes
import os
import socket
import subprocess
import sys

import numpy as np

from oracle import dib_oracle as O
from tests import fused16_oracle as Q
from tests import infonce_oracle as IO
from tests import set_transformer_oracle as STO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- device helpers -------------------------------------------------------------------------------------------------------
def _L():
    from dib_b200 import _lib as L
    return L


def _lib():
    L = _L()
    return L, L.load()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _st():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sms():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


# ---- several processes ----------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_workers(tmp_path, script, world, out, **env):
    """Run ``script`` as ranks 0 .. world - 1 from the repository root (RANK / WORLD_SIZE / MASTER_* set, DIB_ROOT and
    DIB_OUT = ``out`` plus ``env``); every rank must exit 0.  Returns what rank 0 saved to ``out``."""
    path = tmp_path / "worker.py"
    path.write_text(script)
    env = dict(os.environ, DIB_ROOT=ROOT, DIB_OUT=out, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()),
               WORLD_SIZE=str(world), PYTHONPATH=ROOT, **env)
    procs = [subprocess.Popen([sys.executable, str(path)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), cwd=ROOT)
             for r in range(world)]
    try:
        codes = [pr.wait(timeout=600) for pr in procs]
    finally:
        for pr in procs:
            if pr.poll() is None:
                pr.kill()
                pr.wait()
    assert codes == [0] * world, codes
    return dict(np.load(out))


def _compare_fits(a, b, prec):
    """fit at world 2 against world 1: history and weights, fp32 / fp16 bounds of test_gpu_infonce_data_parallel.py"""
    tol_p, tol_h = (1.5e-2, 5e-3) if prec == "fp16" else (2e-4, 2e-4)
    assert set(a) == set(b)
    for k in a:
        if k not in ("params", "graphs"):
            print(f"{prec}: {k} world 2 vs world 1 {rel_err(b[k], a[k]):.3g}")
            np.testing.assert_allclose(b[k], a[k], rtol=tol_h, atol=1e-6, err_msg=k)
    e = rel_err(b["params"], a["params"])
    print(f"{prec}: weights world 2 vs world 1 {e:.3g}")
    assert e < tol_p, e


# ---- DistributedIBNet: the golden cases ---------------------------------------------------------------------------------
LOSS_OF = {"c0_small": ("bce_logits", O.LOSS_BCE_LOGITS), "pendulum_like": ("mse", O.LOSS_MSE),
           "radial_like": ("bce_logits", O.LOSS_BCE_LOGITS), "odd_shapes": ("sparse_ce_logits", O.LOSS_SPARSE_CE_LOGITS)}


def build_model(cfg, precision="fp32", loss="bce_logits", lr=1e-3, seed=0):
    import dib_b200
    m = dib_b200.DistributedIBNet(
        cfg.feature_dimensionalities, cfg.feature_encoder_architecture, cfg.integration_network_architecture,
        cfg.output_dimensionality, use_positional_encoding=cfg.use_positional_encoding,
        number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies,
        activation_fn=cfg.activation_fn, feature_embedding_dimension=cfg.feature_embedding_dimension,
        output_activation_fn=cfg.output_activation_fn, precision=precision, seed=seed, leaky_alpha=cfg.leaky_alpha)
    m.compile(optimizer=dib_b200.Adam(lr), loss=loss, metrics=["accuracy"])
    return m


def load_case(golden_dir, name):
    return O.load_forward_golden(os.path.join(golden_dir, f"ref_forward_{name}.npz"))


def make_labels(rng, loss, B, out):
    if loss == O.LOSS_SPARSE_CE_LOGITS:
        return rng.integers(0, out, size=B).astype(np.float32)
    if loss == O.LOSS_BCE_LOGITS:
        return rng.integers(0, 2, size=(B, out)).astype(np.float32)
    return rng.standard_normal((B, out)).astype(np.float32)


# ---- DistributedIBNet: the C0 model and the boolean circuit -------------------------------------------------------------
def _c0():
    return O.DIBConfig([1] * 16, [128, 128], [256, 256], 1)


def _c0_batch(B, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, 16)).astype(np.float32)
    y = (x[:, 0] * x[:, 1] + np.sin(2 * x[:, 2]) + 0.5 * x[:, 3] > 0).astype(np.float32)[:, None]
    return x, y


def _fit_case():
    """Boolean circuit (data.py:40; SURVEY 8d C1) on a fused-path-eligible model: 10 features, encoders [128,128],
    E=32, integration [256], 4 epochs x 8 steps, beta annealed 1e-3 -> 1e-1 after one pre-training epoch."""
    x, y = O.boolean_circuit_truth_table()
    cfg = O.DIBConfig([1] * 10, [128, 128], [256], 1)
    return x, y, cfg


def _weights(n, seed, hi=50.0):
    """Weights in [0, hi] with zeros and a few exact integers."""
    rng = np.random.default_rng(seed + 77)
    w = rng.uniform(0.0, hi, n).astype(np.float32)
    w[rng.choice(n, max(1, n // 10), replace=False)] = 0.0
    w[:3] = [0.0, 1.0, hi]
    return w


# ---- DistributedIBNet: the 16-bit fused path against tests/fused16_oracle.py ---------------------------------------------
FUSED = {"fp16": "encoders=fused-wgmma-f16 integration=int16-wgmma-f16", "bf16": "encoders=fused-wgmma-bf16 integration=int16-wgmma-bf16"}


def _model(cfg, prec, loss, mask=0, seed=0):
    import dib_b200
    m = dib_b200.DistributedIBNet(
        cfg.feature_dimensionalities, cfg.feature_encoder_architecture, cfg.integration_network_architecture,
        cfg.output_dimensionality, use_positional_encoding=cfg.use_positional_encoding,
        number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies, activation_fn=cfg.activation_fn,
        feature_embedding_dimension=cfg.feature_embedding_dimension, output_activation_fn=cfg.output_activation_fn,
        precision=prec, seed=seed, leaky_alpha=cfg.leaky_alpha, logvar_offset=cfg.logvar_offset,
        kl_loss_exponent=cfg.kl_loss_exponent)
    m.compile(optimizer=dib_b200.Adam(1e-3), loss=loss)
    m.debug_force_unfused(mask)
    return m


def _expect_route(m, prec, n, tail):
    """kernel_info names the route the case means to test: tail in {'dgrad', 'fwd2', None (per-layer GEMMs + a head kernel)}."""
    info = m.kernel_info(n)
    assert FUSED[prec] in info, info
    if tail == "dgrad":
        assert "integration_tail=fwd2-head-dgrad" in info, info
    elif tail == "fwd2":
        assert "integration_tail=fwd2-head" in info and "integration_tail=fwd2-head-dgrad" not in info, info
    else:
        assert "integration_tail" not in info, info


def _params(cfg, seed):
    rng = np.random.default_rng(seed)
    p = O.glorot_uniform_params(cfg, rng)
    return p + (p == 0) * (0.05 * rng.standard_normal(p.size)).astype(np.float32)      # non-zero biases


def _data(cfg, loss, n, seed):
    rng = np.random.default_rng(seed + 1000)
    D, F, E, out = sum(cfg.feature_dimensionalities), cfg.number_features, cfg.feature_embedding_dimension, cfg.output_dimensionality
    x = rng.standard_normal((n, D)).astype(np.float32)
    eps = rng.standard_normal((n, F, E)).astype(np.float32)
    if loss == O.LOSS_SPARSE_CE_LOGITS:
        y = rng.integers(0, out, size=n).astype(np.float32)
    elif loss == O.LOSS_MSE:
        y = rng.standard_normal((n, out)).astype(np.float32)
    else:
        y = (x[:, :1] * x[:, -1:] > 0).astype(np.float32) if out == 1 else rng.integers(0, 2, (n, out)).astype(np.float32)
    return x, y, eps


def _check(what, measured, bound):
    print(f"[fused16-oracle] {what}: {measured:.3e} (bound {bound:.1e})")
    assert measured < bound, (what, measured, bound)


def _stats_err(st, fr, n):
    """KL sums and the loss sum of the step's statistics row against the oracle's, relative."""
    F = len(fr.kl_per_feature)
    kl = np.abs(st[:F] - fr.kl_per_feature * n) / np.abs(fr.kl_per_feature * n)
    lo = abs(st[F] - fr.cache["loss_sum"]) / abs(fr.cache["loss_sum"]) if "loss_sum" in fr.cache else 0.0
    return max(float(kl.max()), float(lo))


# bounds (per-variable max-norm relative unless said otherwise); measured worst values in the comments / DESIGN.md section 2
TOL = {
    # per variable, one step, relu / leaky_relu: bounded by relu-gate flips, not by accumulation (see the notes of
    # test_gpu_fused16_vs_rounding_oracle.py); measured worst 6.3e-2 (fp16, n = 127), 2.1e-2 (fp16, n = 4173), 1.7e-2 (bf16,
    # n = 4173)
    ("grad", "fp16"): 0.1, ("grad", "bf16"): 0.1,
    ("stats", "fp16"): 3e-5, ("stats", "bf16"): 3e-5,        # KL sums and loss sum; measured 8.5e-6 / 7.7e-6
    ("pred", "fp16"): 2e-3, ("pred", "bf16"): 2e-2,          # max-norm relative prediction
    ("emb", "fp16"): 2e-4, ("emb", "bf16"): 2e-3,            # per feature block, u vs the oracle's u; measured 5.0e-5 / 4.1e-4
    ("flip", "fp16"): 1e-2, ("flip", "bf16"): 1e-2,          # fraction of emb16 elements that differ; measured 2.1e-3 / 2.0e-4
    ("tanh", "fp16"): 3e-3, ("tanh", "bf16"): 1.5e-2,        # smooth act': measured 6.5e-4 / 3.5e-3 per variable
    ("rowiso", "fp16"): 3e-3, ("rowiso", "bf16"): 1.5e-2,    # 14 isolated rows; measured 8.4e-4 / 3.3e-3
}


def _grad_case(cfg, prec, loss, n, beta, seed=0, mask=0, tail="dgrad", p=None, label=""):
    p = _params(cfg, seed) if p is None else p
    x, y, eps = _data(cfg, loss, n, seed)
    m = _model(cfg, prec, loss, mask)
    _expect_route(m, prec, n, tail)
    m.set_flat_weights(p)
    m.beta.assign(beta)
    g, st = m.compute_gradients(x, y, eps=eps)
    g, st = g.cpu().numpy().astype(np.float64), st.cpu().numpy().astype(np.float64)
    assert np.isfinite(g).all() and np.isfinite(st).all()
    g_ref, fr = Q.train_grads(cfg, p, x, y, eps, beta, loss, fmt=prec)
    pv = Q.per_variable_errors(cfg, g, g_ref)
    tag = f"{label} {prec} n={n} beta={beta}"
    kind = "tanh" if cfg.activation_fn in ("tanh", "sigmoid", "elu") else "grad"      # smooth act
    _check(f"grad/var {tag} (worst var {int(pv.argmax())})", pv.max(), TOL[(kind, prec)])
    _check(f"stats {tag}", _stats_err(st, fr, n), TOL[("stats", prec)])
    return pv


def _c(F=16, integ=(256, 256), out=1, act="relu", dims=None, **kw):
    out_act = "sigmoid" if kw.pop("probs", False) else None
    return O.DIBConfig(list(dims or [1] * F), [128, 128], list(integ), out, activation_fn=act, output_activation_fn=out_act, **kw)


# ---- DistributedIBNet with losses.InfoNCE -------------------------------------------------------------------------------
# the double-pendulum shape of train.py:116-126 / BASELINE config 3: features [2, 1, 2, 1], out = infonce dim 64,
# output encoder 6 -> PE 30 -> [128, 128] -> 64
CFG = O.DIBConfig([2, 1, 2, 1], [128, 128], [256, 256], 64)
YD, YARCH = 6, [128, 128]


def data(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 6)).astype(np.float32)
    y = np.stack([np.sin(x[:, 0]) * x[:, 1], x[:, 2] * x[:, 3], np.cos(x[:, 4]), x[:, 5] ** 2 - 1, np.tanh(x[:, 0] + x[:, 4]),
                  x[:, 1] * x[:, 5]], -1).astype(np.float32)
    eps = rng.standard_normal((n, 4, 32)).astype(np.float32)
    return x, y, eps


def params(seed):
    rng = np.random.default_rng(seed)
    return IO.glorot(IO.infonce_param_shapes(CFG, YD, YARCH), rng).astype(np.float32)


def temperature_of(similarity):
    return 0.1 if similarity == "cosine" else 1.0


# ---- SetTransformerIBNet ------------------------------------------------------------------------------------------------
def small(L):
    return STO.STConfig(particle_feature_dimensions=3, particle_encoder_arch_spec=[16], bottleneck_dimension=8, number_particles=L,
                        key_dim=12, number_heads=3, number_attention_blocks=2, ff_arch_per_block=[20, 8], final_processing_arch=[12],
                        number_positional_encoding_frequencies=3)


def set_transformer_model(cfg, precision="fp32", seed=0, lr=1e-3, metrics=None, variable=False):
    import dib_b200
    m = dib_b200.SetTransformerIBNet(cfg.particle_feature_dimensions, cfg.particle_encoder_arch_spec, cfg.bottleneck_dimension,
                                     cfg.number_particles, key_dim=cfg.key_dim, number_heads=cfg.number_heads,
                                     number_attention_blocks=cfg.number_attention_blocks, ff_arch_per_block=cfg.ff_arch_per_block,
                                     final_processing_arch=cfg.final_processing_arch,
                                     number_positional_encoding_frequencies=cfg.number_positional_encoding_frequencies,
                                     precision=precision, seed=seed, variable_set_sizes=variable)
    m.compile(optimizer=dib_b200.Adam(lr), loss=dib_b200.losses.BinaryCrossentropy(from_logits=True), metrics=metrics)
    return m


def set_case(cfg, B, seed):
    """B sets of number_particles particles: (params, x, y, eps)"""
    rng = np.random.default_rng(seed)
    p = STO.init_params(cfg, rng)
    x = rng.standard_normal((B, cfg.number_particles, cfg.particle_feature_dimensions)).astype(np.float32)
    eps = rng.standard_normal((B, cfg.number_particles, cfg.bottleneck_dimension)).astype(np.float32)
    y = (rng.random((B, 1)) > 0.5).astype(np.float32)
    return p, x, y, eps


def varlen_set_case(cfg, sizes, seed):
    """set_case of len(sizes) sets, and the sizes as int32: (params, x, y, eps, sizes)"""
    return (*set_case(cfg, len(sizes), seed), np.asarray(sizes, dtype=np.int32))


def _config(**kw):
    """a set-transformer DibConfig for dib_create's checks, with ``kw`` replacing fields; also the arrays it points to"""
    from dib_b200 import _lib
    fd = (ctypes.c_int32 * 1)(3)
    ea = (ctypes.c_int32 * 1)(16)
    ia = (ctypes.c_int32 * 1)(12)
    ff = (ctypes.c_int32 * 2)(20, 8)
    keep = [fd, ea, ia, ff]
    base = dict(abi_version=_lib.ABI_VERSION, number_features=1, feature_dimensionalities=fd, number_encoder_layers=1,
                feature_encoder_architecture=ea, number_integration_layers=1, integration_network_architecture=ia,
                output_dimensionality=1, use_positional_encoding=1, number_positional_encoding_frequencies=3, activation_fn=3,
                leaky_relu_alpha=0.1, feature_embedding_dimension=8, output_activation_fn=0, loss=0, precision=0, max_batch=16,
                integration_kind=1, set_size=7, number_attention_blocks=2, number_heads=3, key_dim=12, number_ff_layers=2,
                ff_architecture=ff, ff_activation_fn=1)
    base.update(kw)
    return _lib.DibConfig(**base), keep
