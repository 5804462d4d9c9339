"""Host-side mirror of the reference's ``models.py`` (PositionalEncoding, DistributedIBNet, the annealing /
compression-matrix / embedding-stash callbacks) on top of the C ABI in include/dib_b200.h.

Same names, constructor arguments and call protocol as /root/reference/models.py:12-223 and the corrected copy
in nb-radial cell 5, so ``train.py``-style drivers and the notebooks' ``model.compile / model.fit`` code run
unchanged with ``import dib_b200.models as models``.  PyTorch is used for device memory, streams and
``torch.distributed`` only; every FLOP of the hot path runs in libdib_b200.so.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import gc
import math
import os
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from . import metrics as _metrics
from . import parallel
from .keras_compat import Adam, InfoNCE, RMSprop, SGD, Callback, History, optimizers, resolve_loss


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.DibError("dib_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _as_numpy_like(ref, t):
    """Return ``t`` in the kind of container ``ref`` was (numpy in -> numpy out, tensor in -> tensor out)."""
    if isinstance(ref, torch.Tensor):
        return t
    return t.detach().cpu().numpy()


def _run_phases(phases, last_exchange=True):
    """Run (launch, exchange) phases eagerly: each launch, then its exchange -- the last phase's only with ``last_exchange``."""
    for k, (launch, exchange) in enumerate(phases):
        launch()
        if exchange is not None and (last_exchange or k < len(phases) - 1):
            exchange()


def _shard_rows(order, b0, b1, rank, world):
    """This rank's rows of the batch [b0, b1) of ``order`` (a permutation, or None for the rows in order) as an index tensor
    or a slice, and their offset in the batch (:func:`parallel.shard_range`)."""
    lo, hi = parallel.shard_range(b1 - b0, rank, world)
    return (order[b0 + lo:b0 + hi] if order is not None else slice(b0 + lo, b0 + hi)), lo


def check_sample_weights(w, n, what="sample_weight"):
    """Host check of the per-sample weights of n rows (sets, for a set transformer): [n] or [n, 1], finite and >= 0.  Returns
    them as a float32 array [n]."""
    a = np.asarray(w)
    if a.dtype.kind not in "biuf":
        raise ValueError(f"{what} must be numeric, got {a.dtype}")
    if a.shape not in ((int(n),), (int(n), 1)):
        raise ValueError(f"{what} has shape {a.shape}; expected one weight per sample, ({int(n)},) or ({int(n)}, 1)")
    a = a.reshape(-1).astype(np.float32)
    if not np.all(np.isfinite(a)) or (a.size and a.min() < 0):
        raise ValueError(f"{what} must be finite and >= 0")
    return a


def check_class_weight(class_weight):
    """[KERAS] ``_make_class_weight_map_fn``: a dict whose keys are exactly 0..C-1.  Returns the float32 table [C]."""
    if not isinstance(class_weight, dict) or not class_weight:
        raise ValueError("class_weight must be a non-empty dict {class index: weight}")
    keys = sorted(class_weight.keys())
    if keys != list(range(len(keys))):
        raise ValueError(f"Expected `class_weight` to be a dict with keys from 0 to one less than the number of classes, "
                         f"found {class_weight}")
    table = np.asarray([float(class_weight[k]) for k in keys], dtype=np.float32)
    if not np.all(np.isfinite(table)) or table.min() < 0:
        raise ValueError("class_weight values must be finite and >= 0")
    return table


def class_weight_classes(y):
    """[KERAS] the class of each row in ``_make_class_weight_map_fn``: argmax over the columns of y [n, k > 1], otherwise y
    reshaped to [n] and cast to an integer, truncating (float labels 1.7 -> 1).  Non-finite labels map to -1."""
    a = np.asarray(y)
    if a.ndim > 2:
        raise ValueError("class_weight is not supported for 3+ dimensional targets")
    if a.ndim == 2 and a.shape[1] > 1:
        return a.argmax(axis=1).astype(np.int64)
    v = a.reshape(-1).astype(np.float64)
    return np.where(np.isfinite(v), np.trunc(np.where(np.isfinite(v), v, 0.0)), -1).astype(np.int64)


def class_weight_rows(y, class_weight, sample_weight=None):
    """Host statement of the row weights ``fit(..., class_weight=, sample_weight=)`` trains with (dib_class_weight_rows
    computes them on the device): table[class of row i], times sample_weight[i] when given, in float32.  Labels outside
    0..C-1 raise ValueError."""
    table = check_class_weight(class_weight)
    cls = class_weight_classes(y)
    bad = (cls < 0) | (cls >= table.size)
    if bad.any():
        raise ValueError(f"class_weight: label {np.asarray(y).reshape(len(cls), -1)[bad][0].tolist()} of row "
                         f"{int(np.flatnonzero(bad)[0])} has no class in 0..{table.size - 1}")
    w = table[cls]
    if sample_weight is not None:
        w = check_sample_weights(sample_weight, len(cls)) * w
    return w


def check_weighted_loss(loss_kind, output_dimensionality, class_weight=False):
    """Refuse sample / class weights where the compiled loss cannot take them: losses.InfoNCE and the external loss (the
    caller owns the loss), and class_weight with MSE or a multi-output BCE (no class label to map)."""
    if loss_kind in ("infonce", "external"):
        raise ValueError(f"the {loss_kind!r} loss takes no sample_weight / class_weight")
    if class_weight and (loss_kind == "mse" or (loss_kind != "sparse_ce_logits" and int(output_dimensionality) != 1)):
        raise ValueError("class_weight needs a class label per row: sparse categorical cross-entropy, or binary "
                         f"cross-entropy with one output (compiled loss {loss_kind!r}, {int(output_dimensionality)} outputs)")


class PositionalEncoding:
    """models.py:12-23.  Kept for API parity; inside DistributedIBNet the encoding is fused into the first-layer
    operand by the library.  Calling it directly is a convenience (plain torch ops, not the hot path)."""

    def __init__(self, frequencies):
        self.frequencies = list(frequencies)

    def __call__(self, inputs):
        freqs = [int(f) for f in self.frequencies]
        if freqs != [2 ** k for k in range(1, len(freqs) + 1)]:
            raise NotImplementedError("the library's positional encoding uses the reference's frequencies 2**arange(1, n)")
        _require_cuda()
        t = torch.as_tensor(inputs, dtype=torch.float32)
        dev = t.device if t.is_cuda else torch.device("cuda", torch.cuda.current_device())
        x = t.to(dev).reshape(-1, t.shape[-1]).contiguous()
        out = torch.empty(x.shape[0], x.shape[1] * (len(freqs) + 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().dib_positional_encoding(_lib.ptr(x), x.shape[0], x.shape[1], len(freqs) + 1, _lib.ptr(out),
                                                           _stream()))
        return _as_numpy_like(inputs, out.reshape(*t.shape[:-1], out.shape[-1]))

    call = __call__


class _Beta:
    """``tf.Variable(1., dtype=tf.float32, trainable=False)`` surface used by the callbacks (models.py:86,148,177)."""

    def __init__(self, device):
        self._host = np.float32(1.0)
        self._dev = torch.ones(1, dtype=torch.float32, device=device)

    def assign(self, value):
        self._host = np.float32(value)
        self._dev.fill_(float(self._host))
        return self

    def value(self):
        return self._host

    numpy = value

    def __float__(self):
        return float(self._host)

    def __array__(self, dtype=None, copy=None):
        return np.asarray(self._host, dtype=dtype)

    # arithmetic the reference's drivers do with the variable: ``kl_loss / model.beta`` (train.py:214),
    # ``self.beta * tensor`` (models.py:118), ``beta * 2.0`` -- delegate to the float32 host value
    def _other(self, o):
        return o.to(torch.float32) if isinstance(o, torch.Tensor) else o

    def __mul__(self, o): return float(self._host) * self._other(o)
    __rmul__ = __mul__
    def __truediv__(self, o): return float(self._host) / self._other(o)
    def __rtruediv__(self, o): return self._other(o) / float(self._host)
    def __add__(self, o): return float(self._host) + self._other(o)
    __radd__ = __add__
    def __sub__(self, o): return float(self._host) - self._other(o)
    def __rsub__(self, o): return self._other(o) - float(self._host)
    def __neg__(self): return -float(self._host)
    def __repr__(self): return f"<beta {float(self._host)!r}>"


class _Network:
    """A view of one Dense stack inside the flat parameter buffer (model.feature_encoders[i] /
    model.integration_network): ``.weights`` are torch views [W, b, W, b, ...] in Keras order."""

    def __init__(self, model, var_slice):
        self._model = model
        self._vars = var_slice

    @property
    def weights(self):
        return [self._model._var_view(i) for i in self._vars]

    trainable_variables = weights

    def get_weights(self):
        return [w.detach().cpu().numpy() for w in self.weights]


class _FeatureEncoder(_Network):
    """model.feature_encoders[i]: deterministic [n, d_i] -> [n, 2E] (mu || logvar), the contract used by
    visualization.py:31, utils.py:38 and StashEmbeddingsCallback.  Runs dib_encode_feature."""

    def __init__(self, model, index, var_slice):
        super().__init__(model, var_slice)
        self.index = index

    def __call__(self, x_i, training=None):
        return _as_numpy_like(x_i, self._model._encode_feature(self.index, x_i))


class _IntegrationNetwork(_Network):
    """model.integration_network (models.py:84), or the set transformer of :class:`SetTransformerIBNet`: embeddings
    [n, width] (width = F * E, or number_particles * E for the set transformer) -> [n, out].  Direct calls are rare (the fused
    step never materialises this boundary); they run dib_integration_forward on the model's precision path."""

    def __init__(self, model, var_slice, width):
        super().__init__(model, var_slice)
        self._width = width

    def __call__(self, emb, training=None, set_sizes=None):
        m = self._model
        with torch.cuda.device(m.device):
            e, sd = m._integration_inputs(emb, set_sizes, self._width)
            n = e.shape[0]
            m._ensure_handle(n)
            m._bind_set_sizes(sd)
            out = torch.empty(n, m.output_dimensionality, dtype=torch.float32, device=m.device)
            _lib.check(m._lib.dib_integration_forward(m._handle, _lib.ptr(m._params), _lib.ptr(e), n, _lib.ptr(out),
                                                      _lib.ptr(m._workspace), _stream()))
        return _as_numpy_like(emb[0] if isinstance(emb, list) and emb else emb, out)


class _OutputEncoder(_Network):
    """model.output_encoder of a model compiled with ``losses.InfoNCE`` (train.py:186-193): deterministic
    [n, y_dimensionality] -> [n, output_dimensionality].  Runs dib_output_encoder_forward."""

    def __call__(self, y, training=None):
        m = self._model
        with torch.cuda.device(m.device):
            t = m._targets(y)
            n = t.shape[0]
            m._ensure_handle(n)
            out = torch.empty(n, m.output_dimensionality, dtype=torch.float32, device=m.device)
            _lib.check(m._lib.dib_output_encoder_forward(m._handle, _lib.ptr(m._params), _lib.ptr(t), n, _lib.ptr(out),
                                                         _lib.ptr(m._workspace), _stream()))
        return _as_numpy_like(y, out)


def infonce_epoch_batches(n, batch_size):
    """The training batches of one InfoNCE epoch (train.py:222-231): InfoNCE needs full, equal batches, so an epoch is
    floor(n / batch_size) consecutive slices [b0, b1) of that epoch's permutation and the remainder is dropped."""
    n, batch_size = int(n), int(batch_size)
    if n < batch_size:
        raise ValueError(f"InfoNCE needs at least one full batch: {n} samples < batch_size {batch_size}")
    return [(k * batch_size, (k + 1) * batch_size) for k in range(n // batch_size)]


def infonce_validation_batches(n, batch_size):
    """The validation batches of InfoNCE (train.py:233-234: ``repeat().shuffle().batch(B).take(n // B + 1)``):
    floor(n / batch_size) + 1 full batches of positions into the validation permutation, repeated end to end, so the
    last batch wraps around.  Returns an int64 array [batches, batch_size]."""
    n, batch_size = int(n), int(batch_size)
    if n < 1:
        raise ValueError("empty validation set")
    nb = n // batch_size + 1
    return np.arange(nb * batch_size, dtype=np.int64).reshape(nb, batch_size) % n


class DistributedIBNet:
    """Distributed IB model where each feature is passed through its own probabilistic encoder MLP
    (models.py:26-123; ``dropout_rate``/``training`` from nb-radial cell 5).

    Custom-step variants of the same front end (keyword-only; SURVEY 8f3):
      ``feature_encoder_architecture='simple'`` -- nb-bool cell 4's SimpleEncoder for every feature (two trainable (1,1)
        constants mu_scaling = 1, logvar = -3; needs d_i == feature_embedding_dimension, no positional encoding);
      ``logvar_offset`` -- constant added to every encoder's log-variance (nb-particle cell 8, -3 there);
      ``kl_loss_exponent`` / ``kl_loss_scale`` -- nonlinear IB ``beta * scale * (sum_i KL_i) ** exponent`` (nb-chaos cell 10);
      ``model.encode`` / ``model.encoder_gradients`` -- encoder-only steps for a caller-owned downstream network
        (nb-particle's shared particle encoder + set transformer: see :class:`SharedParticleEncoder`).

    Extra keyword-only arguments (not in the reference): ``device``, ``seed`` (weight init + noise stream),
    ``precision`` ('fp32' exact-FMA parity path | 'tf32' tf32 wgmma GEMMs | 'fp16' / 'bf16' fused 16-bit-operand
    wgmma kernels with fp32 accumulation; ``model.kernel_info()`` says what a handle actually runs), ``process_group``
    (data-parallel group; defaults to the WORLD group when torch.distributed is initialised), ``leaky_alpha``.
    """

    variable_set_sizes = False         # SetTransformerIBNet(variable_set_sizes=True): inputs carry per-set sizes

    def __init__(self,
                 feature_dimensionalities: Sequence[int],
                 feature_encoder_architecture: Sequence[int],
                 integration_network_architecture: Sequence[int],
                 output_dimensionality: int,
                 use_positional_encoding: bool = True,
                 number_positional_encoding_frequencies: int = 5,
                 activation_fn: Optional[str] = 'relu',
                 feature_embedding_dimension: int = 32,
                 output_activation_fn: Optional[str] = None,
                 dropout_rate: float = 0.,
                 *, device=None, seed: int = 0, precision: str = 'fp32', process_group=None,
                 leaky_alpha: float = 0.2, logvar_offset: float = 0., kl_loss_exponent: float = 1.,
                 kl_loss_scale: float = 1.):
        _require_cuda()
        if not (0.0 <= float(dropout_rate) < 1.0):
            raise ValueError("dropout_rate must be in [0, 1)")
        self.dropout_rate = float(dropout_rate)       # nb-radial cell 5: Dropout after every hidden encoder Dense (train steps only)
        if activation_fn not in _lib.ACTIVATIONS or output_activation_fn not in _lib.ACTIVATIONS:
            raise ValueError(f"unsupported activation {activation_fn!r}/{output_activation_fn!r}")
        if precision not in _lib.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISIONS)}, got {precision!r}")
        self.feature_dimensionalities = [int(d) for d in feature_dimensionalities]
        self.number_features = len(self.feature_dimensionalities)
        self.encoder_kind = "simple" if isinstance(feature_encoder_architecture, str) else "mlp"
        if self.encoder_kind == "simple":
            if feature_encoder_architecture != "simple":
                raise ValueError("feature_encoder_architecture must be a list of widths or 'simple'")
            feature_encoder_architecture, use_positional_encoding = [], False
        self.logvar_offset = float(logvar_offset)
        self.kl_loss_exponent = float(kl_loss_exponent)
        self.kl_loss_scale = float(kl_loss_scale)
        self.feature_encoder_architecture = [int(h) for h in feature_encoder_architecture]
        self.integration_network_architecture = [int(h) for h in integration_network_architecture]
        self.output_dimensionality = int(output_dimensionality)
        self.use_positional_encoding = bool(use_positional_encoding)
        self.number_positional_encoding_frequencies = int(number_positional_encoding_frequencies)
        self.activation_fn = activation_fn
        self.output_activation_fn = output_activation_fn
        self.feature_embedding_dimension = int(feature_embedding_dimension)
        self.leaky_alpha = float(leaky_alpha)
        self.precision = precision
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.seed = int(seed)
        self.noise_seed = int(seed)
        self.process_group = process_group
        self.stop_training = False

        self._lib = _lib.load()
        self._loss_kind = "bce_logits"
        self._infonce = None               # the compiled losses.InfoNCE: its output encoder is part of the parameters
        self._handle = None
        self._handle_key = None
        self._workspace = None
        self._query_layout()

        with torch.cuda.device(self.device):
            self.beta = _Beta(self.device)                                   # models.py:86
            self._params = torch.zeros(self._P, dtype=torch.float32, device=self.device)
            self._init_glorot_uniform()
            self._gradstats = torch.zeros(self._P + self.number_features + 3, dtype=torch.float32, device=self.device)
            self._m = torch.zeros_like(self._params)
            self._v = torch.zeros_like(self._params)
            self._lr_dev = torch.full((1,), 1e-3, dtype=torch.float32, device=self.device)
            self._step_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._epoch_acc = torch.zeros(self.number_features + 4, dtype=torch.float32, device=self.device)
            self._epoch_tail = torch.zeros(0, dtype=torch.float64, device=self.device)    # compiled metrics' epoch sums
        self._train_step_count = 0
        # ---- CUDA-graph replay of the train step (launch-bound small batches; fewer host calls per step at any size)
        env = os.environ.get("DIB_CUDA_GRAPH", "auto").lower()
        self.use_cuda_graph = env not in ("0", "off", "false", "no")
        self._graphs = {}                  # (n, global_batch, sample_offset, world) -> captured step
        self._graph_seen = {}              # eager executions per key before capture (lazy one-time setup must be done)
        self._graph_failed = False
        self._noise_step_dev = None        # int32 device mirror of _train_step_count (Philox step word inside graphs)
        self._step_dev_active = False
        self._step_dev_dirty = False       # _train_step_count moved outside a graph replay: refill the device mirror
        self._replayed_launches = 0        # kernels launched by graph replays (dib_launch_count only sees eager launches)
        self._inference_calls = 0          # fresh noise per un-seeded inference call (tf.random.normal, models.py:108)
        self.optimizer = None
        self.compiled_metrics_names = []
        self._metric_entries = []          # metrics.CompiledMetric per compiled metric, in history order
        self._tail_len = 0                 # floats of the metric tail behind the F + 3 statistics
        self.losses = []
        self.metrics_values = {}
        n_enc_vars = 2 if self.encoder_kind == "simple" else 2 * (len(self.feature_encoder_architecture) + 1)
        self.feature_encoders = [                                            # models.py:79
            _FeatureEncoder(self, i, range(i * n_enc_vars, (i + 1) * n_enc_vars)) for i in range(self.number_features)]
        self._n_model_vars = len(self._var_off)
        self.integration_network = _IntegrationNetwork(                      # models.py:84
            self, range(self.number_features * n_enc_vars, self._n_model_vars),
            self.number_features * self.feature_embedding_dimension)
        self.output_encoder = None                                           # losses.InfoNCE: train.py:186-193
        self._p_enc = int(self._var_off[self.number_features * n_enc_vars])  # first integration-network parameter

    # ------------------------------------------------------------------ library handle / buffers
    def _config(self, max_batch):
        F = self.number_features
        self._c_fd = (ctypes.c_int32 * F)(*self.feature_dimensionalities)
        L, Li = len(self.feature_encoder_architecture), len(self.integration_network_architecture)
        self._c_ea = (ctypes.c_int32 * max(L, 1))(*self.feature_encoder_architecture)
        self._c_ia = (ctypes.c_int32 * max(Li, 1))(*self.integration_network_architecture)
        nce = self._infonce
        y_arch = nce.y_encoder_architecture if nce is not None else []
        self._c_ya = (ctypes.c_int32 * max(len(y_arch), 1))(*y_arch)
        from .utils import SIMILARITY_TYPES
        return _lib.DibConfig(
            abi_version=_lib.ABI_VERSION, number_features=F, feature_dimensionalities=self._c_fd,
            number_encoder_layers=L, feature_encoder_architecture=self._c_ea,
            number_integration_layers=Li, integration_network_architecture=self._c_ia,
            output_dimensionality=self.output_dimensionality,
            use_positional_encoding=int(self.use_positional_encoding),
            number_positional_encoding_frequencies=self.number_positional_encoding_frequencies,
            activation_fn=_lib.ACTIVATIONS[self.activation_fn], leaky_relu_alpha=self.leaky_alpha,
            feature_embedding_dimension=self.feature_embedding_dimension,
            output_activation_fn=_lib.ACTIVATIONS[self.output_activation_fn],
            loss=_lib.LOSSES[self._loss_kind], precision=_lib.PRECISIONS[self.precision], max_batch=int(max_batch),
            logvar_offset=self.logvar_offset, kl_loss_exponent=self.kl_loss_exponent, kl_loss_scale=self.kl_loss_scale,
            encoder_kind=_lib.ENCODER_KINDS[self.encoder_kind], dropout_rate=self.dropout_rate,
            y_dimensionality=nce.y_dimensionality if nce is not None else 0, number_y_encoder_layers=len(y_arch),
            y_encoder_architecture=self._c_ya, infonce_similarity=SIMILARITY_TYPES[nce.similarity] if nce is not None else 0,
            infonce_temperature=nce.temperature if nce is not None else 1.0)

    def _query_layout(self):
        with torch.cuda.device(self.device):
            h = ctypes.c_void_p()
            cfg = self._config(1)
            _lib.check(self._lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)))
            try:
                self._P = int(self._lib.dib_param_count(h))
                nv = self._lib.dib_param_layout(h, None, None, None, 0)
                offs, rows, cols = (ctypes.c_int64 * nv)(), (ctypes.c_int32 * nv)(), (ctypes.c_int32 * nv)()
                assert self._lib.dib_param_layout(h, offs, rows, cols, nv) == nv
                self._var_off, self._var_rows, self._var_cols = list(offs), list(rows), list(cols)
            finally:
                self._lib.dib_destroy(h)

    def _ensure_handle(self, n):
        key = (self._loss_kind, self.precision, self._infonce.spec() if self._infonce is not None else None,
               _metrics.signature(self._metric_entries))
        if self._handle is not None and self._handle_key == key and n <= self._max_batch:
            return
        self._release_handle()
        max_batch = max(int(n), 1)
        with torch.cuda.device(self.device):
            h = ctypes.c_void_p()
            cfg = self._config(max_batch)
            _lib.check(self._lib.dib_create(ctypes.byref(cfg), ctypes.byref(h)))
            self._handle, self._handle_key, self._max_batch = h, key, max_batch
            self._graphs.clear(); self._graph_seen.clear()       # captured launches point into the old workspace
            self._step_dev_active = False
            if getattr(self, "_force_unfused", 0):
                _lib.check(self._lib.dib_debug_force_unfused(h, int(self._force_unfused)))
            if self._tail_len:
                specs, count = _metrics.library_specs(self._metric_entries)
                _lib.check(self._lib.dib_set_metrics(h, specs, count))
            assert int(self._lib.dib_stats_count(h)) == self._stats_count()
            nbytes = int(self._lib.dib_workspace_bytes(h))
            self._workspace = None
            self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            assert self._workspace.data_ptr() % 256 == 0

    def kernel_info(self, batch_hint=1):
        """What the library runs for this model: precision, kernel families, operand / accumulator types."""
        with torch.cuda.device(self.device):
            self._ensure_handle(max(int(batch_hint), 1))
            buf = ctypes.create_string_buffer(512)
            if self._lib.dib_model_info(self._handle, buf, len(buf)) < 0:
                raise _lib.DibError(self._lib.dib_last_error().decode())
        return buf.value.decode()

    def _release_handle(self):
        if getattr(self, "_handle", None) is not None:
            torch.cuda.synchronize(self.device)
            self._lib.dib_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._release_handle()
        except Exception:
            pass

    def _var_view(self, i):
        off, r, c = self._var_off[i], self._var_rows[i], self._var_cols[i]
        v = self._params[off:off + max(r, 1) * c]
        return v.view(r, c) if r > 0 else v

    def _init_glorot_uniform(self):
        """Keras Dense defaults: kernel glorot_uniform, bias zeros (third-party behaviour; RNG stream is ours)."""
        self._params.copy_(self._glorot_flat())

    def _param_inits(self):
        """The initializer of every variable in flat order: ('glorot', fan_in, fan_out), 'zeros', 'ones' or a constant."""
        n_simple = 2 * self.number_features if self.encoder_kind == "simple" else 0
        inits = []
        for k, (r, c) in enumerate(zip(self._var_rows, self._var_cols)):
            if k < n_simple:                 # nb-bool cell 4: mu_scaling = ones, logvar = -3 * ones
                inits.append(1.0 if k % 2 == 0 else -3.0)
            else:
                inits.append(("glorot", r, c) if r > 0 else "zeros")
        return inits

    def _glorot_flat(self):
        """The flat weights :meth:`_param_inits` describes; glorot_uniform draws one generator seeded by ``seed`` in flat
        order (RNG stream is ours)."""
        g = torch.Generator(device="cpu")
        g.manual_seed(self.seed)
        flat = torch.zeros(self._P, dtype=torch.float32)
        for off, r, c, init in zip(self._var_off, self._var_rows, self._var_cols, self._param_inits()):
            size = max(r, 1) * c
            if isinstance(init, tuple):
                lim = math.sqrt(6.0 / (init[1] + init[2]))
                flat[off:off + size] = (torch.rand(size, generator=g) * 2 - 1) * lim
            elif init != "zeros":
                flat[off:off + size] = 1.0 if init == "ones" else init
        return flat

    def _set_output_encoder(self, nce):
        """Lay the output encoder of ``nce`` (a losses.InfoNCE, or None) out after the model's variables: the flat buffer,
        the optimizer slots and [grads || stats] grow or shrink, the model's weights and slots are kept, and the output
        encoder starts from the glorot-uniform values a fresh model of the joint layout gets from ``seed``."""
        old_spec = self._infonce.spec() if self._infonce is not None else None
        new_spec = nce.spec() if nce is not None else None
        self._infonce = nce
        if old_spec == new_spec:
            return
        keep = self._var_off[self._n_model_vars] if self._n_model_vars < len(self._var_off) else self._P
        self._release_handle()
        self._graphs.clear(); self._graph_seen.clear()
        self._query_layout()
        with torch.cuda.device(self.device):
            params = self._glorot_flat().to(self.device)
            params[:keep] = self._params[:keep]
            m, v = torch.zeros_like(params), torch.zeros_like(params)
            m[:keep], v[:keep] = self._m[:keep], self._v[:keep]
            self._params, self._m, self._v = params, m, v
            self._gradstats = torch.zeros(self._P + self._stats_count(), dtype=torch.float32, device=self.device)
        self._staging = None
        self.output_encoder = (_OutputEncoder(self, range(self._n_model_vars, len(self._var_off)))
                               if nce is not None else None)

    # ------------------------------------------------------------------ Keras-like variable access
    @property
    def trainable_variables(self):
        return [self._var_view(i) for i in range(len(self._var_off))]

    trainable_weights = trainable_variables
    weights = trainable_variables

    def get_weights(self):
        return [v.detach().cpu().numpy() for v in self.trainable_variables]

    def set_weights(self, weights):
        vs = self.trainable_variables
        if len(weights) != len(vs):
            raise ValueError(f"expected {len(vs)} arrays, got {len(weights)}")
        for v, w in zip(vs, weights):
            v.copy_(torch.as_tensor(np.asarray(w), dtype=torch.float32).view(v.shape))

    def get_flat_weights(self):
        return self._params.detach().cpu().numpy()

    def set_flat_weights(self, flat):
        self._params.copy_(torch.as_tensor(np.asarray(flat), dtype=torch.float32))

    def count_params(self):
        return self._P

    def build(self, input_shape):
        assert input_shape[-1] == sum(self.feature_dimensionalities)       # models.py:89

    def _stats_count(self):
        """Floats of the statistics vector: [KL sums (F) | task loss | accuracy | n] and the compiled metrics' tail."""
        return self.number_features + 3 + self._tail_len

    # ------------------------------------------------------------------ data helpers
    def _to_device(self, a, cols=None):
        if a is None:
            return None
        t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
        t = t.to(device=self.device, dtype=torch.float32, non_blocking=True)
        if cols is not None:
            t = t.reshape(t.shape[0], cols) if cols > 0 else t.reshape(t.shape[0])
        return t.contiguous()

    def _y_cols(self):
        if self._infonce is not None:
            return self._infonce.y_dimensionality
        return 0 if self._loss_kind == "sparse_ce_logits" else self.output_dimensionality

    def _targets(self, y):
        """y on the device as [n, _y_cols()]; an InfoNCE model checks the width (it sizes the output encoder)."""
        if self._infonce is not None:
            shape = tuple(y.shape)
            if len(shape) not in (1, 2) or (shape[-1] if len(shape) == 2 else 1) != self._infonce.y_dimensionality:
                raise ValueError(f"y has shape {shape}; the InfoNCE output encoder takes [n, {self._infonce.y_dimensionality}]")
        return self._to_device(y, self._y_cols())

    def _inputs(self, x):
        """Model inputs on the device: (x [n, sum d_i], per-set sizes or None -- see SetTransformerIBNet)."""
        return self._to_device(x, sum(self.feature_dimensionalities)), None

    def _integration_inputs(self, emb, set_sizes, width):
        if set_sizes is not None:
            raise ValueError("set_sizes is for SetTransformerIBNet(variable_set_sizes=True)")
        return self._to_device(emb, width), None

    def _bind_set_sizes(self, sizes):
        """Point the handle at the int32 device sizes of the sets of the following library calls (variable set sizes)."""
        if sizes is not None:
            _lib.check(self._lib.dib_set_set_sizes_device(self._handle, _lib.ptr(sizes)))

    def _bind_sample_weights(self, weights):
        """Point the handle at the fp32 device weights of the rows of the following library calls (None: unweighted)."""
        _lib.check(self._lib.dib_set_sample_weights_device(self._handle, _lib.ptr(weights)))

    def _sample_weights(self, sample_weight, n, what="sample_weight"):
        """sample_weight checked on the host (one read of a device tensor), then as float32 [n] on the device; None stays
        None."""
        if sample_weight is None:
            return None
        check_weighted_loss(self._loss_kind, self.output_dimensionality)
        t = sample_weight if isinstance(sample_weight, torch.Tensor) else None
        host = check_sample_weights(t.detach().cpu().numpy() if t is not None else sample_weight, n, what)
        if t is not None:
            return t.to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        return torch.from_numpy(host).to(self.device)

    def _row_weights(self, y, yd, sample_weight, class_weight, n):
        """The training weights of n rows: sample_weight, or with class_weight the Keras class map of y (labels checked on
        the host, the rows mapped on the device by dib_class_weight_rows) times sample_weight.  None when neither is given."""
        wd = self._sample_weights(sample_weight, n)
        if class_weight is None:
            return wd
        check_weighted_loss(self._loss_kind, self.output_dimensionality, class_weight=True)
        yh = y.detach().cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y)
        table = check_class_weight(class_weight)
        class_weight_rows(yh, class_weight)                     # the label check, before any device work
        td = torch.from_numpy(table).to(self.device)
        out = torch.empty(n, dtype=torch.float32, device=self.device)
        _lib.check(self._lib.dib_class_weight_rows(_lib.ptr(yd), n, yd.shape[1] if yd.dim() == 2 else 0, _lib.ptr(td),
                                                   table.size, _lib.ptr(wd), _lib.ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ compute entry points
    def _forward(self, x, y, eps, step, sample_offset, want_pred=True, want_emb=False, stats_out=None, sizes=None,
                 weights=None):
        n = x.shape[0]
        self._ensure_handle(n)
        self._bind_set_sizes(sizes)
        self._bind_sample_weights(weights)
        pred = torch.empty(n, self.output_dimensionality, dtype=torch.float32, device=self.device) if want_pred else None
        emb = torch.empty(n, self.number_features * self.feature_embedding_dimension, dtype=torch.float32,
                          device=self.device) if want_emb else None
        stats = stats_out if stats_out is not None else torch.empty(self._stats_count(), dtype=torch.float32,
                                                                    device=self.device)
        _lib.check(self._lib.dib_forward(
            self._handle, _lib.ptr(self._params), _lib.ptr(x), _lib.ptr(y), n, _lib.ptr(self.beta._dev), _lib.ptr(eps),
            self.noise_seed, int(step) & 0xFFFFFFFF, int(sample_offset), _lib.ptr(pred), _lib.ptr(emb), _lib.ptr(stats),
            _lib.ptr(self._workspace), _stream()))
        return pred, emb, stats

    def _encoder_rows(self, i, x_i):
        """x_i on the device as encoder i's input rows [rows, d_i], and the batch size the handle needs for them."""
        t = self._to_device(x_i, self.feature_dimensionalities[i])
        return t, t.shape[0]

    def _encode_feature(self, i, x_i):
        t, batch = self._encoder_rows(i, x_i)
        n = t.shape[0]
        self._ensure_handle(batch)
        out = torch.empty(n, 2 * self.feature_embedding_dimension, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.dib_encode_feature(self._handle, _lib.ptr(self._params), i, _lib.ptr(t), n,
                                                    _lib.ptr(out), _lib.ptr(self._workspace), _stream()))
        return out

    def compression_matrices(self, x, row_index=None, want=("mu_logvar", "dist", "comp")):
        """All features at once (dib_compression_matrices; visualization.py:14-35 loops over features in Python):
        rows ``row_index[i]`` of ``x`` -> encoder i -> Bhattacharyya -> exp(-D).  ``row_index``: [F, n] integer array or
        None (= all rows of x for every feature).  Returns a dict of device tensors for the names in ``want``:
        mu_logvar [F, n, 2E], dist [F, n, n], comp [F, n, n]."""
        t = self._to_device(x, sum(self.feature_dimensionalities))
        F, E = self.number_features, self.feature_embedding_dimension
        if row_index is None:
            n, idx = t.shape[0], None
        else:
            idx = row_index if isinstance(row_index, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(row_index))
            idx = idx.to(device=self.device, dtype=torch.int32).contiguous()
            if idx.dim() != 2 or idx.shape[0] != F:
                raise ValueError("row_index must have shape [number_features, n]")
            n = idx.shape[1]
        self._ensure_handle(max(n, 1))
        out = {}
        if "mu_logvar" in want:
            out["mu_logvar"] = torch.empty(F, n, 2 * E, dtype=torch.float32, device=self.device)
        if "dist" in want:
            out["dist"] = torch.empty(F, n, n, dtype=torch.float32, device=self.device)
        if "comp" in want:
            out["comp"] = torch.empty(F, n, n, dtype=torch.float32, device=self.device)
        opt = lambda k: _lib.ptr(out[k]) if k in out else None
        with torch.cuda.device(self.device):
            _lib.check(self._lib.dib_compression_matrices(self._handle, _lib.ptr(self._params), _lib.ptr(t), t.shape[0],
                                                          _lib.ptr(idx) if idx is not None else None, n, opt("mu_logvar"),
                                                          opt("dist"), opt("comp"), _lib.ptr(self._workspace), _stream()))
        return out

    def _set_device_step(self, on):
        """Philox step word from the device mirror of _train_step_count (graph replay) or by value (everything else)."""
        if on == self._step_dev_active and self._handle is not None and not (on and self._step_dev_dirty):
            return
        if on:
            self._step_dev_dirty = False
            if self._noise_step_dev is None:
                self._noise_step_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._noise_step_dev.fill_(int(self._train_step_count) & 0x7FFFFFFF)
        _lib.check(self._lib.dib_set_noise_step_device(self._handle, _lib.ptr(self._noise_step_dev) if on else None))
        self._step_dev_active = on

    def _step_phases(self, x, y, global_batch, eps, sample_offset, step, device_step=False, training=True, stats=None,
                     sizes=None, weights=None):
        """The train step of one batch as an ordered list of (launch, exchange): ``exchange`` is the collective that has to
        follow ``launch`` -- the all-gather of e_all or lse_all, or the all-reduce of self._gradstats = [grads (P) || stats
        (F+3)] -- and None where there is none, which is everywhere with one process.  ``step`` is the Philox step word.

        dib_train_step, the all-reduce, the optimizer update; losses.InfoNCE(negatives='global') on more than one rank splits
        dib_train_step into its three shard phases with the two all-gathers between them (DESIGN.md section 7).  With
        ``device_step`` (graph capture) the optimizer phase also advances the device noise step; ``training`` and ``stats``
        (default the stats of self._gradstats) go to the InfoNCE shard forward and lse; ``sizes`` are the set sizes of a
        variable-size set transformer, and ``weights`` the rows' sample weights (or None), bound to the handle right before
        its train step."""
        n, P, group = x.shape[0], self._P, self.process_group
        self._ensure_handle(n)
        world, rank = parallel.world_and_rank(group)
        stats = self._gradstats[P:] if stats is None else stats
        gather = (lambda t: lambda: parallel.all_gather_rows_(t, group)) if world > 1 else (lambda t: None)
        reduce = (lambda: parallel.allreduce_sum_(self._gradstats, group)) if world > 1 else None

        def update():
            self._adam()
            if device_step:
                self._noise_step_dev.add_(1)

        if self._infonce is not None and world > 1:
            n_global, row_offset = self._infonce_shard(n, global_batch, world, rank)
            e_all, lse_all = self._infonce_buffers(n_global)
            phases = [
                (lambda: self._infonce_forward(x, y, e_all, n_global, row_offset, eps, step, sample_offset, training),
                 gather(e_all)),
                (lambda: self._infonce_lse(n, e_all, lse_all, n_global, row_offset, stats), gather(lse_all)),
                (lambda: self._infonce_backward(x, e_all, lse_all, n_global, row_offset, eps, step, sample_offset), reduce)]
        else:
            def train_step():
                self._bind_set_sizes(sizes)
                self._bind_sample_weights(weights)
                _lib.check(self._lib.dib_train_step(
                    self._handle, _lib.ptr(self._params), _lib.ptr(x), _lib.ptr(y), n, _lib.ptr(self.beta._dev),
                    1.0 / float(global_batch), _lib.ptr(eps), self.noise_seed, int(step) & 0xFFFFFFFF,
                    int(sample_offset), _lib.ptr(self._gradstats), _lib.ptr(self._gradstats[P:]), _lib.ptr(self._workspace),
                    _stream()))
            phases = [(train_step, reduce)]
        return phases + [(update, None)]

    def _backward(self, x, y, global_batch, eps=None, sample_offset=0, step=None, device_step=False, sizes=None, weights=None):
        """Forward + reverse mode into self._gradstats = [grads (P) || stats (F+3)] of this rank: the step's phases up to
        the all-reduce."""
        st = 0 if device_step else (self._train_step_count if step is None else step)
        phases = self._step_phases(x, y, global_batch, eps, sample_offset, st, device_step, sizes=sizes, weights=weights)
        self._set_device_step(device_step)
        _run_phases(phases[:-1], last_exchange=False)

    # ------------------------------------------------------------------ InfoNCE with global negatives on several ranks
    def _check_infonce_world(self, nce, batch_size=None):
        """Refuse, before any device work or collective, what data-parallel InfoNCE cannot do."""
        world, _ = parallel.world_and_rank(self.process_group)
        if world == 1:
            return
        if nce.negatives is None:
            raise NotImplementedError(
                "losses.InfoNCE couples every row of the global batch, so with more than one rank the negatives of a row must "
                "be chosen: compile with losses.InfoNCE(..., negatives='global') to all-gather the embeddings of the global "
                "batch and train on exactly the one-process loss")
        if batch_size is not None and int(batch_size) % world:
            raise ValueError(f"InfoNCE with negatives='global' needs equal shards: batch_size {batch_size} is not a multiple "
                             f"of the {world} ranks")

    def _infonce_shard(self, n, global_batch, world, rank):
        """(n_global, row_offset) of this rank's n rows: equal shards, rank r owns rows [r n, (r + 1) n)."""
        self._check_infonce_world(self._infonce)
        if global_batch is not None and int(global_batch) != world * n:
            raise ValueError(f"InfoNCE with negatives='global' needs equal shards: global_batch {global_batch} != "
                             f"{world} ranks x {n} rows")
        return world * n, rank * n

    def _infonce_buffers(self, n_global):
        """e_all [n_global, 2 d] = (e1 || e2) per row and lse_all [n_global, 2] = (r, c) per row."""
        d = self.output_dimensionality
        return (torch.empty(n_global, 2 * d, dtype=torch.float32, device=self.device),
                torch.empty(n_global, 2, dtype=torch.float32, device=self.device))

    def _infonce_forward(self, x, y, e_all, n_global, row_offset, eps, step, sample_offset, training):
        _lib.check(self._lib.dib_infonce_shard_forward(
            self._handle, _lib.ptr(self._params), _lib.ptr(x), _lib.ptr(y), x.shape[0], int(training), _lib.ptr(eps),
            self.noise_seed, int(step) & 0xFFFFFFFF, int(sample_offset), _lib.ptr(e_all), n_global, row_offset,
            _lib.ptr(self._workspace), _stream()))

    def _infonce_lse(self, n, e_all, lse_all, n_global, row_offset, stats_out):
        _lib.check(self._lib.dib_infonce_shard_lse(self._handle, _lib.ptr(e_all), n_global, row_offset, n, _lib.ptr(lse_all),
                                                   _lib.ptr(stats_out), _lib.ptr(self._workspace), _stream()))

    def _infonce_backward(self, x, e_all, lse_all, n_global, row_offset, eps, step, sample_offset):
        _lib.check(self._lib.dib_infonce_shard_backward(
            self._handle, _lib.ptr(self._params), _lib.ptr(x), x.shape[0], _lib.ptr(self.beta._dev), _lib.ptr(eps),
            self.noise_seed, int(step) & 0xFFFFFFFF, int(sample_offset), _lib.ptr(e_all), _lib.ptr(lse_all), n_global,
            row_offset, _lib.ptr(self._gradstats), _lib.ptr(self._workspace), _stream()))

    def apply_gradients(self, flat_grads):
        """optimizer.apply_gradients(zip(grads, model.trainable_variables)) of the custom loops (train.py:217-219,
        nb-bool cell 6): one Keras-Adam update of the flat parameter buffer with caller-supplied gradients."""
        g = torch.as_tensor(flat_grads, dtype=torch.float32).to(self.device).contiguous()
        if g.numel() != self._P:
            raise ValueError(f"expected {self._P} gradient values, got {g.numel()}")
        self._sync_lr()
        with torch.cuda.device(self.device):
            self._optimizer_update(g)
        self._train_step_count += 1
        self._step_dev_dirty = True

    def _optimizer_update(self, grads):
        """One dense update of the flat parameter buffer by the compiled optimizer (Adam: dib_adam_step; SGD / RMSprop:
        dib_optimizer_step); the two slot buffers are Adam's m / v, SGD's velocity, RMSprop's mean square / momentum."""
        opt = self.optimizer
        if isinstance(opt, Adam):
            _lib.check(self._lib.dib_adam_step(
                _lib.ptr(self._params), _lib.ptr(grads), _lib.ptr(self._m), _lib.ptr(self._v), self._P,
                _lib.ptr(self._lr_dev), _lib.ptr(self._step_dev), opt.beta_1, opt.beta_2, opt.epsilon, _stream()))
        else:
            h0, h1, h2 = opt.hyper()
            _lib.check(self._lib.dib_optimizer_step(
                opt.kind, _lib.ptr(self._params), _lib.ptr(grads), _lib.ptr(self._m), _lib.ptr(self._v), self._P,
                _lib.ptr(self._lr_dev), _lib.ptr(self._step_dev), h0, h1, h2, _stream()))

    def _adam(self):
        self._optimizer_update(self._gradstats)

    def _train_step(self, x, y, global_batch, eps=None, sample_offset=0, sizes=None, weights=None):
        """backward, one flat all-reduce of [grads || stats] over the data-parallel group, Keras-Adam.  Replayed from
        CUDA graphs once a (batch size, offset, weighted or not, compiled metrics) combination has run eagerly twice; the set sizes of a
        variable-size set transformer and the sample weights are data, not part of that key."""
        P = self._P
        world, _ = parallel.world_and_rank(self.process_group)
        key = (int(x.shape[0]), int(global_batch), int(sample_offset), world, _metrics.signature(self._metric_entries),
               weights is not None)
        if self.use_cuda_graph and not self._graph_failed and eps is None and x.shape[0] > 0:
            g = self._graphs.get(key)
            if g is None and self._graph_seen.get(key, 0) >= 2:
                g = self._capture_step(key, with_sizes=sizes is not None)
            if g is not None:
                return self._replay_step(g, x, y, sizes, weights)
            self._graph_seen[key] = self._graph_seen.get(key, 0) + 1
        phases = self._step_phases(x, y, global_batch, eps, sample_offset, self._train_step_count, sizes=sizes,
                                   weights=weights)
        self._set_device_step(False)
        _run_phases(phases)
        self._train_step_count += 1
        self._step_dev_dirty = True
        return self._gradstats[P:]

    # ------------------------------------------------------------------ CUDA-graph replay of the step
    def _capture_step(self, key, with_sizes=False):
        """Capture the step for one (n, global_batch, sample_offset, world, compiled metrics, weighted) into CUDA graphs: one graph per run of phases
        between two collectives, each kept with the exchange that follows it.  Single GPU: ONE graph (forward + backward +
        optimizer + noise-step increment); plain data parallel: two (backward | optimizer); InfoNCE with global negatives: four
        (the three shard phases | optimizer), e_all / lse_all kept with the graphs.  Inputs are copied into static buffers
        before each replay (and, ``with_sizes``, the set sizes into a third one; weighted, the sample weights into a fourth); beta, learning rate, the optimizer step and
        the Philox step are device scalars, so nothing by-value changes between replays."""
        n, global_batch, sample_offset, world, _, weighted = key
        D = sum(self.feature_dimensionalities)
        yc = self._y_cols()
        try:
            with torch.cuda.device(self.device):
                gx = torch.zeros(n, D, dtype=torch.float32, device=self.device)
                gy = torch.zeros((n, yc) if yc > 0 else (n,), dtype=torch.float32, device=self.device)
                gs = torch.ones(n, dtype=torch.int32, device=self.device) if with_sizes else None
                gw = torch.ones(n, dtype=torch.float32, device=self.device) if weighted else None
                phases = self._step_phases(gx, gy, global_batch, None, sample_offset, 0, device_step=True, sizes=gs,
                                           weights=gw)
                self._set_device_step(True)
                torch.cuda.synchronize(self.device)
                keep = [t.clone() for t in (self._params, self._m, self._v, self._step_dev, self._noise_step_dev)]
                graphs, run = [], []
                launches0 = int(self._lib.dib_launch_count())
                # a garbage collection inside the capture could finalize a dead model, whose synchronize and dib_destroy
                # would invalidate the capture
                gc_on = gc.isenabled()
                gc.disable()
                try:
                    for k, (launch, exchange) in enumerate(phases):
                        run.append(launch)
                        if exchange is not None or k == len(phases) - 1:
                            g = torch.cuda.CUDAGraph()
                            with torch.cuda.graph(g):
                                for fn in run:
                                    fn()
                            graphs.append((g, exchange))
                            run = []
                finally:
                    if gc_on:
                        gc.enable()
                torch.cuda.synchronize(self.device)
                # capture does not execute, but be safe against any eager side effect: restore the optimizer state
                for t, k in zip((self._params, self._m, self._v, self._step_dev, self._noise_step_dev), keep):
                    t.copy_(k)
        except Exception as e:       # noqa: BLE001 -- an unsupported capture falls back to eager launches, loudly
            import warnings
            warnings.warn(f"CUDA-graph capture of the train step failed ({e!r}); continuing with eager launches")
            self._graph_failed = True
            self._set_device_step(False)
            return None
        g = dict(graphs=graphs, x=gx, y=gy, sizes=gs, weights=gw, launches=int(self._lib.dib_launch_count()) - launches0)
        self._graphs[key] = g
        return g

    def _replay_step(self, g, x, y, sizes=None, weights=None):
        P = self._P
        if not self._step_dev_active or self._step_dev_dirty:
            self._set_device_step(True)
        self._replayed_launches += g["launches"]
        g["x"].copy_(x.reshape(g["x"].shape), non_blocking=True)
        g["y"].copy_(y.reshape(g["y"].shape), non_blocking=True)
        if g["sizes"] is not None:
            g["sizes"].copy_(sizes, non_blocking=True)
        if g["weights"] is not None:
            g["weights"].copy_(weights, non_blocking=True)
        for graph, exchange in g["graphs"]:
            graph.replay()
            if exchange is not None:
                exchange()
        self._train_step_count += 1
        return self._gradstats[P:]

    def compute_gradients(self, x, y, eps=None, global_batch=None, sample_offset=0, step=None, sample_weight=None):
        """GradientTape-style access (nb-bool cell 6 / train.py:201-220 custom loops): returns
        (flat gradient of task + beta*sum KL w.r.t. trainable_variables, statistics vector) as device tensors.
        ``sample_weight`` [n] weights each row's task loss (Keras SUM_OVER_BATCH_SIZE: sum_i w_i l_i / global_batch)."""
        with torch.cuda.device(self.device):
            xd, sd = self._inputs(x)
            yd = self._targets(y)
            wd = self._sample_weights(sample_weight, xd.shape[0])
            e = self._to_device(eps) if eps is not None else None
            if not global_batch:            # InfoNCE on several ranks: every rank passes its equal shard of the global batch
                nce_world = parallel.world_and_rank(self.process_group)[0] if self._infonce is not None else 1
                global_batch = max(xd.shape[0] * nce_world, 1)
            self._backward(xd, yd, global_batch, e, sample_offset, step, sizes=sd, weights=wd)
            return self._gradstats[:self._P].clone(), self._gradstats[self._P:].clone()

    # ------------------------------------------------------------------ encoder-only custom steps (SURVEY 8f3)
    def encode(self, x, eps=None, step=None, sample_offset=0):
        """Every feature encoder + reparameterisation, without the integration network (nb-particle cell 8's
        ``particle_encoder`` front end): returns (emb [n, F*E] = mu + exp(logvar/2) eps, KL_i batch means [F]) as device
        tensors.  Noise as in ``__call__``: explicit ``eps``, Philox keyed by ``step``, or a fresh draw."""
        self._refuse_tail_metrics("encode")
        with torch.cuda.device(self.device):
            xd = self._to_device(x, sum(self.feature_dimensionalities))
            e = self._to_device(eps) if eps is not None else None
            n = xd.shape[0]
            self._ensure_handle(n)
            st = self._inference_step() if step is None else step
            emb = torch.empty(n, self.number_features * self.feature_embedding_dimension, dtype=torch.float32, device=self.device)
            stats = torch.empty(self.number_features + 3, dtype=torch.float32, device=self.device)
            _lib.check(self._lib.dib_encoders_forward(
                self._handle, _lib.ptr(self._params), _lib.ptr(xd), n, _lib.ptr(e), self.noise_seed, int(st) & 0xFFFFFFFF,
                int(sample_offset), _lib.ptr(emb), _lib.ptr(stats), _lib.ptr(self._workspace), _stream()))
            return emb, stats[:self.number_features] / max(n, 1)

    def encoder_gradients(self, x, d_emb, global_batch=None, eps=None, step=None, sample_offset=0):
        """Reverse mode of :meth:`encode` for a caller-owned downstream network: ``d_emb`` [n, F*E] is d(caller's loss)/d(emb)
        (already carrying the caller's batch scaling); the IB term beta * scale * (sum KL)^p, with KL means over
        ``global_batch`` rows (default n), is added here.  Returns (flat gradient [P] -- integration entries are zero --,
        statistics vector).  Pass the same ``eps`` / ``step`` as the ``encode`` call it differentiates."""
        self._refuse_tail_metrics("encoder_gradients")
        with torch.cuda.device(self.device):
            xd = self._to_device(x, sum(self.feature_dimensionalities))
            gd = self._to_device(d_emb, self.number_features * self.feature_embedding_dimension)
            e = self._to_device(eps) if eps is not None else None
            n = xd.shape[0]
            self._ensure_handle(n)
            st = self._train_step_count if step is None else step
            P = self._P
            _lib.check(self._lib.dib_encoders_backward(
                self._handle, _lib.ptr(self._params), _lib.ptr(xd), _lib.ptr(gd), n, _lib.ptr(self.beta._dev),
                1.0 / float(global_batch or max(n, 1)), _lib.ptr(e), self.noise_seed, int(st) & 0xFFFFFFFF, int(sample_offset),
                _lib.ptr(self._gradstats), _lib.ptr(self._gradstats[P:]), _lib.ptr(self._workspace), _stream()))
            return self._gradstats[:P].clone(), self._gradstats[P:].clone()

    def debug_force_unfused(self, on=True, batch_hint=1):
        """Bring-up switch: keep the tensor-core mode on the reference kernels (fused-vs-unfused comparisons).

        ``on`` is a bit mask (``True`` = 1): 1 = unfused encoders, 2 = fp32-storage TF32 integration network, 4 = no fused
        integration tail (per-layer 16-bit GEMMs plus a head kernel), 8 = the generic head kernel even when out = 1, 16 = the
        fused tail without its dgrad stages (separate dgrad launches in the backward)."""
        self._force_unfused = int(on)
        if self._handle is not None:
            _lib.check(self._lib.dib_debug_force_unfused(self._handle, int(on)))

    def epoch_permutation(self, epoch, n):
        """The shuffle Model.fit applies in ``epoch`` (our RNG stream; Keras' own is irreproducible)."""
        gen = torch.Generator(device=self.device)
        gen.manual_seed((self.seed << 20) + epoch)
        return torch.randperm(n, generator=gen, device=self.device)

    def _zero_epoch(self):
        self._epoch_acc.zero_()
        self._epoch_tail.zero_()

    def _metrics_update(self, stats):
        _lib.check(self._lib.dib_metrics_update_ex(_lib.ptr(stats), _lib.ptr(self.beta._dev), _lib.ptr(self._epoch_acc),
                                                   self.number_features, self.kl_loss_exponent, self.kl_loss_scale, _stream()))
        if self._tail_len:
            F = self.number_features
            _lib.check(self._lib.dib_metrics_update_tail(_lib.ptr(stats[F + 3:]), _lib.ptr(self._epoch_tail), self._tail_len,
                                                         _stream()))

    def _metric_logs(self, acc_sum, n, tail, prefix=""):
        """{prefix + name: value} of the compiled metrics in history order: the accuracy slot (acc_sum / n) and the tail's."""
        vals = _metrics.metric_values(self._metric_entries, tail) if self._tail_len else {}
        return {prefix + e.name: (float(acc_sum / n) if not e.in_tail else vals[e.name]) for e in self._metric_entries}

    def _read_epoch_logs(self, prefix=""):
        F = self.number_features
        a = self._epoch_acc.detach().cpu().numpy().astype(np.float64)       # one D2H per epoch
        tail = self._epoch_tail.detach().cpu().numpy() if self._tail_len else None
        n, nb = max(a[F + 2], 1.0), max(a[F + 3], 1.0)
        logs = {prefix + "loss": float(a[F] / n)}
        logs.update(self._metric_logs(a[F + 1], n, tail, prefix))
        for i in range(F):
            logs[f"{prefix}KL{i}"] = float(a[i] / nb)                        # add_metric mean over batches (models.py:115)
        logs[prefix + "beta"] = float(self.beta.value())                     # models.py:121
        return logs

    # ------------------------------------------------------------------ Keras-like public surface
    def _inference_step(self):
        """Philox 'step' word of an un-seeded inference call: bit 31 marks inference (training steps count from 0),
        bit 30 separates it from the validation passes of fit, the low bits count calls -- every call draws fresh
        noise like tf.random.normal at models.py:108 does."""
        self._inference_calls += 1
        return (3 << 30) | (self._inference_calls & 0x3FFFFFFF)

    def __call__(self, inputs, training=None, eps=None, step=None, sample_offset=0):
        """models.py:96-123.  Returns the prediction; ``model.losses`` then holds [beta * sum_i KL_i] and
        ``model.metrics_values`` the KL{i}/beta metrics, as add_loss/add_metric leave them in the reference.
        Noise: explicit ``eps`` [n, F, E], or Philox keyed by ``step`` (reproducible), or -- default -- a fresh draw
        on every call."""
        with torch.cuda.device(self.device):
            x, sd = self._inputs(inputs)
            e = self._to_device(eps) if eps is not None else None
            st = self._inference_step() if step is None else step
            pred, _, stats = self._forward(x, None, e, st, sample_offset, sizes=sd)
            n = x.shape[0]
            kl = stats[:self.number_features] / max(n, 1)
            self.losses = [self.beta._dev[0] * self.kl_loss_scale * kl.sum() ** self.kl_loss_exponent]
            self._last_kl = kl
            self.metrics_values = {"beta": self.beta.value()}
        return _as_numpy_like(inputs[0] if isinstance(inputs, (list, tuple)) and inputs else inputs, pred)

    call = __call__

    def compile(self, optimizer='adam', loss=None, metrics=None, weighted_metrics=None, **_):
        """train.py:138-142, and Keras' compiled metrics: ``metrics`` / ``weighted_metrics`` take 'accuracy' (its own
        statistics slot, as before), the strings 'binary_accuracy', 'sparse_categorical_accuracy', 'mse' /
        'mean_squared_error', 'mae' / 'mean_absolute_error', 'binary_crossentropy', 'sparse_categorical_crossentropy'
        (Keras' functions as written: from_logits=False) and the objects of :mod:`dib_b200.metrics` (AUC, Precision,
        Recall with one output).  ``weighted_metrics`` weight each row by the step's sample weight; a metric in both lists
        gets the ``weighted_`` prefix on its weighted copy.  History keys are the names as written (objects: ``name``) and
        their ``val_`` twins; see :mod:`dib_b200.metrics` for the semantics and the refusals."""
        new_opt = optimizers.get(optimizer)
        kind = resolve_loss(loss)
        if kind == "infonce":
            if metrics or weighted_metrics:
                raise ValueError("losses.InfoNCE has no accuracy: compile it without metrics (train.py:180-289 tracks none)")
            if self.output_activation_fn is not None:
                raise ValueError("losses.InfoNCE needs output_activation_fn=None: the prediction is the InfoNCE embedding "
                                 "(train.py:117)")
            self._check_infonce_world(loss)
        entries = _metrics.compile_metrics(metrics, weighted_metrics, kind, self.output_dimensionality,
                                           self.output_activation_fn)
        if new_opt is not self.optimizer:        # a fresh Keras optimizer has fresh slots and iteration count
            self._m.zero_(); self._v.zero_(); self._step_dev.zero_()
        self.optimizer = new_opt
        self._loss_kind = kind
        self._set_output_encoder(loss if kind == "infonce" else None)
        self._set_metric_entries(entries)
        self._lr_host = None
        self._sync_lr()

    def _set_metric_entries(self, entries):
        """The compiled metrics: history names, the tail length, and the device buffers whose size depends on it."""
        self._metric_entries = entries
        self.compiled_metrics_names = [e.name for e in entries]
        tail = _metrics.tail_length(entries)
        if tail != self._tail_len:
            self._tail_len = tail
            with torch.cuda.device(self.device):
                self._gradstats = torch.zeros(self._P + self._stats_count(), dtype=torch.float32, device=self.device)
                self._epoch_tail = torch.zeros(tail, dtype=torch.float64, device=self.device)

    def _refuse_tail_metrics(self, what):
        if self._tail_len:
            raise ValueError(f"{what} is an encoder-only step and computes no compiled metrics: compile the model without "
                             "metrics other than 'accuracy' to use it")

    def _sync_lr(self):
        """Device copy of optimizer.learning_rate (the step kernels read it from memory so that a schedule needs no re-capture);
        refreshed only when the host value changed -- one fill kernel per step otherwise."""
        lr = float(self.optimizer.learning_rate)
        if lr != getattr(self, "_lr_host", None):
            self._lr_dev.fill_(lr)
            self._lr_host = lr

    def train_on_batch(self, x, y, sample_weight=None, class_weight=None, return_dict=True, sync=True):
        """One optimizer step on a (host or device) batch; ``sample_weight`` / ``class_weight`` weight the rows' task loss
        as in :meth:`fit`.

        ``sync=True`` (Keras behaviour): returns the batch metrics (dict, or the scalar loss) -- forces the D2H read.
        ``sync=False``: returns a :class:`PendingBatchResult`; host batches are staged through a copy stream with two
        device slots and the metrics are copied to pinned memory asynchronously, so the H2D copy of call k+1 overlaps
        the compute of call k.  ``result.get()`` (or the next sync point) yields the same dict."""
        if self.optimizer is None:
            raise RuntimeError("call compile() first")
        with torch.cuda.device(self.device):
            self._sync_lr()
            D = sum(self.feature_dimensionalities)
            world, rank = parallel.world_and_rank(self.process_group)
            host_x = not (isinstance(x, torch.Tensor) and x.is_cuda)
            if sync or not host_x or self.variable_set_sizes:      # sized sets are not staged through the copy stream
                (xd, sd), yd = self._inputs(x), self._targets(y)
                n = xd.shape[0]
                wd = self._row_weights(y, yd, sample_weight, class_weight, n)
                stats = self._train_step(xd, yd, global_batch=n * world, sample_offset=rank * n, sizes=sd, weights=wd)
                res = PendingBatchResult(self, stats.detach().clone() if not sync else stats, None, None)
            else:
                w = None
                if sample_weight is not None or class_weight is not None:      # checked and mapped on the host, staged as x, y
                    n = len(x)
                    check_weighted_loss(self._loss_kind, self.output_dimensionality, class_weight is not None)
                    w = (class_weight_rows(np.asarray(y), class_weight, sample_weight) if class_weight is not None
                         else check_sample_weights(sample_weight.detach().cpu().numpy()
                                                   if isinstance(sample_weight, torch.Tensor) else sample_weight, n))
                xd, yd, wd, slot = self._stage_async(x, y, D, w)
                n = xd.shape[0]
                stats = self._train_step(xd, yd, global_batch=n * world, sample_offset=rank * n, weights=wd)
                st = self._staging
                st["done"][slot].record(torch.cuda.current_stream())          # slot may be overwritten after this
                hi = (st["k"] - 1) % len(st["stats_host"])
                if st["pending"][hi] is not None:
                    st["pending"][hi].get()                                   # its pinned buffer is about to be reused
                host = st["stats_host"][hi]
                host.copy_(stats, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
                res = PendingBatchResult(self, None, host, ev)
                st["pending"][hi] = res
        if not sync:
            return res
        out = res.get()
        return out if return_dict else out["loss"]

    def _stage_async(self, x, y, D, w=None):
        """H2D of a host batch (and its float32 row weights w, or None) on the copy stream into one of two device slots; the
        compute stream waits on it."""
        xt = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        yt = y if isinstance(y, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32))
        n, yc = xt.shape[0], self._y_cols()
        st = getattr(self, "_staging", None)
        if st is None or st["n"] != n or st["stats_host"][0].numel() != self._stats_count():
            st = dict(n=n, k=0, stream=torch.cuda.Stream(device=self.device),
                      x=[torch.empty(n, D, dtype=torch.float32, device=self.device) for _ in range(2)],
                      y=[torch.empty((n, yc) if yc > 0 else (n,), dtype=torch.float32, device=self.device) for _ in range(2)],
                      w=[torch.empty(n, dtype=torch.float32, device=self.device) for _ in range(2)],
                      done=[torch.cuda.Event() for _ in range(2)], copied=[torch.cuda.Event() for _ in range(2)],
                      stats_host=[torch.empty(self._stats_count(), dtype=torch.float32).pin_memory() for _ in range(8)],
                      pending=[None] * 8, used=[False, False])
            self._staging = st
        slot = st["k"] % 2
        st["k"] += 1
        cs = st["stream"]
        if st["used"][slot]:
            cs.wait_event(st["done"][slot])                   # the step that read this slot two calls ago has finished
        with torch.cuda.stream(cs):
            st["x"][slot].copy_(xt.reshape(n, D), non_blocking=True)
            st["y"][slot].copy_(yt.reshape(st["y"][slot].shape), non_blocking=True)
            if w is not None:
                st["w"][slot].copy_(torch.from_numpy(w), non_blocking=True)
            st["copied"][slot].record(cs)
        torch.cuda.current_stream().wait_event(st["copied"][slot])
        st["used"][slot] = True
        return st["x"][slot], st["y"][slot], (st["w"][slot] if w is not None else None), slot

    def fit(self, x=None, y=None, batch_size=None, epochs=1, verbose='auto', callbacks=None, validation_data=None,
            shuffle=True, initial_epoch=0, class_weight=None, sample_weight=None, **_):
        """Keras ``Model.fit`` mechanics around the fused step (train.py:157-166, nb-radial cell 10): per epoch
        on_epoch_begin -> shuffled consecutive batches incl. a short last one -> running means -> validation pass
        (noise sampled, train.py:264-265) -> on_epoch_end; returns a History whose ``.history`` has the keys
        loss, accuracy, KL{i}, beta and their val_ twins.

        Data-parallel: with torch.distributed initialised every rank passes the SAME x, y; each global batch is
        split into contiguous row ranges per rank, so the result does not depend on the number of GPUs.

        ``sample_weight`` [N] and ``class_weight`` {0: w_0, ..., C-1: w_{C-1}} weight each row's task loss as Keras does
        [KERAS]: loss = sum_i w_i l_i / batch size + beta * sum KL (the KL term and ``accuracy`` are unweighted); class_weight
        maps a row to its class by argmax of a one-hot y or by the truncated integer label, and multiplies sample_weight
        when both are given.  ``validation_data=(x_val, y_val, w_val)`` weights the validation loss by w_val; class_weight
        applies to training only.

        Compiled with ``losses.InfoNCE`` this runs train.py:180-289's InfoNCE training, which needs full, equal batches:
        an epoch is floor(N / batch_size) batches of the epoch permutation (the remainder is dropped; N < batch_size is an
        error) and validation takes floor(Nv / batch_size) + 1 full batches from the repeated validation permutation.
        History keys are loss (= InfoNCE + beta * sum KL, so ``loss - beta * sum KL`` is the InfoNCE term), KL{i}, beta and
        their val_ twins.  beta follows the annealing callback's on_epoch_begin, i.e. it is set before an epoch's first
        step; the reference's custom loop assigns it after that step (train.py:245-250), one step late.  With more than one
        rank it needs ``losses.InfoNCE(..., negatives='global')`` and a batch_size that is a multiple of the number of ranks:
        every rank then trains on its equal shard of the same global batches and the result is the one-process result."""
        if self.optimizer is None:
            raise RuntimeError("call compile() first")
        batch_size = 32 if batch_size is None else int(batch_size)
        world, rank = parallel.world_and_rank(self.process_group)
        if self._infonce is not None:
            self._check_infonce_world(self._infonce, batch_size)
        with torch.cuda.device(self.device):
            (xd, sd), yd = self._inputs(x), self._targets(y)
            N = xd.shape[0]
            plan = self._batch_plan(N, batch_size)
            xv = yv = sv = wv = None
            if validation_data is not None:
                (xv, sv), yv = self._inputs(validation_data[0]), self._targets(validation_data[1])
                if len(validation_data) > 2:
                    wv = self._sample_weights(validation_data[2], xv.shape[0], "validation sample_weight")
            wd = self._row_weights(y, yd, sample_weight, class_weight, N)
            history = History()
            cbs = list(callbacks or []) + [history]
            for cb in cbs:
                cb.set_model(self) if hasattr(cb, "set_model") else setattr(cb, "model", self)
            self.history = history
            self.stop_training = False
            for cb in cbs:
                getattr(cb, "on_train_begin", lambda logs=None: None)()
            for epoch in range(initial_epoch, epochs):
                for cb in cbs:
                    cb.on_epoch_begin(epoch, logs=None)                      # beta annealing lives here
                self._sync_lr()
                order = self.epoch_permutation(epoch, N) if shuffle else None
                self._zero_epoch()
                for b0, b1 in plan:
                    idx, lo = _shard_rows(order, b0, b1, rank, world)
                    self._metrics_update(self._train_step(xd[idx], yd[idx], global_batch=b1 - b0, sample_offset=lo,
                                                          sizes=None if sd is None else sd[idx],
                                                          weights=None if wd is None else wd[idx]))
                logs = self._read_epoch_logs()
                if xv is not None:
                    logs.update(self._evaluate_into_logs(xv, yv, *self._validation_plan(xv.shape[0], batch_size, epoch),
                                                         2 ** 31 + epoch, sv, wv))
                if verbose not in (False, 0) and rank == 0:          # 'auto' -> 1 like Keras outside notebooks
                    print(f"Epoch {epoch + 1}/{epochs} - " + " - ".join(
                        f"{k}: {v:.4g}" for k, v in logs.items() if not k.removeprefix('val_').startswith('KL')))
                for cb in cbs:
                    cb.on_epoch_end(epoch, logs)
                if self.stop_training:
                    break
            for cb in cbs:
                getattr(cb, "on_train_end", lambda logs=None: None)()
        return history

    def _batch_plan(self, n, batch_size):
        """The [b0, b1) batches of one pass over n rows: full ones for InfoNCE (:func:`infonce_epoch_batches`), otherwise
        consecutive batches with a short last one."""
        if self._infonce is not None:
            return infonce_epoch_batches(n, batch_size)
        return [(b0, min(b0 + batch_size, n)) for b0 in range(0, n, batch_size)]

    def _validation_plan(self, n, batch_size, perm_key):
        """(batches, row order) of a validation pass over n rows.  InfoNCE (train.py:233-234): floor(n / B) + 1 full batches
        drawn from the repeated validation permutation of ``perm_key`` (:func:`infonce_validation_batches`); otherwise the
        rows in order (order None)."""
        if self._infonce is None:
            return self._batch_plan(n, batch_size), None
        pos = torch.from_numpy(infonce_validation_batches(n, batch_size)).to(self.device)
        order = self.validation_permutation(perm_key, n)[pos].reshape(-1)
        return self._batch_plan(order.shape[0], batch_size), order

    def _evaluate_into_logs(self, xv, yv, plan, order, step, sv=None, wv=None):
        """Validation logs of the batches ``plan`` of rows ``order`` (see :func:`_shard_rows`), noise keyed by (step, the
        row's position in ``order``): every rank runs the forward of its shard of a batch -- InfoNCE with more than one rank
        the first two phases of the step, without training -- and the statistics are summed over the ranks."""
        world, rank = parallel.world_and_rank(self.process_group)
        self._zero_epoch()
        stats = torch.empty(self._stats_count(), dtype=torch.float32, device=self.device)
        for b0, b1 in plan:
            idx, lo = _shard_rows(order, b0, b1, rank, world)
            if self._infonce is not None and world > 1:
                phases = self._step_phases(xv[idx], yv[idx], b1 - b0, None, b0 + lo, step, training=False, stats=stats)
                _run_phases(phases[:2], last_exchange=False)
            else:
                self._forward(xv[idx], yv[idx], None, step, b0 + lo, want_pred=False, stats_out=stats,
                              sizes=None if sv is None else sv[idx], weights=None if wv is None else wv[idx])
            parallel.allreduce_sum_(stats, self.process_group)
            self._metrics_update(stats)
        return self._read_epoch_logs(prefix="val_")

    def validation_permutation(self, key, n):
        """The shuffle of the InfoNCE validation set for ``key`` (the epoch in fit; our RNG stream)."""
        gen = torch.Generator(device=self.device)
        gen.manual_seed((self.seed << 20) + (1 << 19) + int(key))
        return torch.randperm(n, generator=gen, device=self.device)

    def evaluate(self, x, y, batch_size=32, return_dict=True, sample_weight=None, **_):
        """Loss (task weighted by ``sample_weight`` [n] when given, as in :meth:`fit`), accuracy and KL of one pass over x."""
        with torch.cuda.device(self.device):
            self._inference_calls += 1           # a fresh noise draw per evaluate() call
            key = (1 << 29) | (self._inference_calls & 0x1FFFFFFF)
            if self._infonce is not None:
                self._check_infonce_world(self._infonce, batch_size)
            (xv, sv), yv = self._inputs(x), self._targets(y)
            wv = self._sample_weights(sample_weight, xv.shape[0])
            step = key if self._infonce is not None else 2 ** 31 + key
            logs = self._evaluate_into_logs(xv, yv, *self._validation_plan(xv.shape[0], int(batch_size), key), step, sv, wv)
        logs = {k[len("val_"):]: v for k, v in logs.items()}
        return logs if return_dict else [logs["loss"]] + [logs[m] for m in self.compiled_metrics_names]

    def predict(self, x, batch_size=32, **_):
        outs = []
        n = len(x)
        st = self._inference_step()              # one noise stream per predict(); rows keyed by their global index
        for b0 in range(0, n, int(batch_size)):
            xb = x[b0:b0 + int(batch_size)]
            o = self(xb, training=False, step=st, sample_offset=b0)
            outs.append(o if isinstance(x, torch.Tensor) else np.asarray(o))
        return torch.cat(outs) if isinstance(x, torch.Tensor) else np.concatenate(outs)


class PendingBatchResult:
    """Metrics of one ``train_on_batch(..., sync=False)`` call; ``get()`` waits for the asynchronous D2H copy."""

    def __init__(self, model, stats_dev, stats_host, event):
        self._m, self._dev, self._host, self._ev = model, stats_dev, stats_host, event
        self._beta = float(model.beta.value())
        self._out = None

    def get(self):
        if self._out is None:
            if self._ev is not None:
                self._ev.synchronize()
                s = self._host.numpy().astype(np.float64)            # copy out of the pinned buffer
            else:
                s = self._dev.detach().cpu().numpy().astype(np.float64)
            F = self._m.number_features
            nn = max(s[F + 2], 1.0)
            m = self._m
            ib = self._beta * m.kl_loss_scale * (s[:F].sum() / nn) ** m.kl_loss_exponent      # models.py:118 / nb-chaos
            out = {"loss": float(s[F] / nn + ib), "accuracy": float(s[F + 1] / nn)}
            if m._tail_len:                              # the batch's compiled metrics (Keras reset_metrics=True)
                out.update(_metrics.metric_values(m._metric_entries, s[F + 3:F + 3 + m._tail_len]))
            for i in range(F):
                out[f"KL{i}"] = float(s[i] / nn)
            self._out = out
        return self._out

    def __getitem__(self, k):
        return self.get()[k]


class InfoBottleneckAnnealingCallback(Callback):
    """Callback to logarithmically increase beta during training (models.py:125-149).  The schedule is
    evaluated in float32 exactly like the tf ops there:
        beta = exp(log b0 + float32(max(epoch - n_pre, 0)) / n_anneal * (log b1 - log b0))."""

    def __init__(self, beta_start, beta_end, number_pretraining_epochs, number_annealing_epochs):
        super().__init__()
        self.beta_start = beta_start
        self.beta_end = beta_end
        self.number_pretraining_epochs = number_pretraining_epochs
        self.number_annealing_epochs = number_annealing_epochs

    def beta_at(self, epoch):
        f = np.float32
        frac = f(max(epoch - self.number_pretraining_epochs, 0)) / f(self.number_annealing_epochs)
        lo, hi = np.log(f(self.beta_start)), np.log(f(self.beta_end))
        return f(np.exp(lo + frac * (hi - lo)))

    def on_epoch_begin(self, epoch, logs=None):
        self.model.beta.assign(self.beta_at(epoch))


class SaveCompressionMatricesCallback(Callback):
    """Callback to save compression scheme matrices during training (models.py:152-186; the intended behaviour is
    the inline copy at train.py:251-261 -- the shipped on_epoch_end raises NameError).  For every feature: pick
    <=128 rows as visualization.py:17-28 does, encoder forward, Bhattacharyya matrix, exp(-D) (all features in one
    device call, dib_compression_matrices).  The reference renders a PNG with matplotlib, which is not available
    here; the numeric artefact is saved as ``feature_{i}_log10beta_{x:.3f}.npz`` (same stem) and kept in
    ``self.matrices``."""

    def __init__(self, save_frequency, x_processed, x_raw, outdir, max_number_to_display=128, seed=0):
        super().__init__()
        self.save_frequency = save_frequency
        self.x_processed = x_processed
        self.x_raw = x_raw
        self.outdir = outdir
        self.max_number_to_display = max_number_to_display
        self.rng = np.random.default_rng(seed)
        self.matrices = []

    def on_epoch_end(self, epoch, logs=None):
        if (epoch % self.save_frequency) != 0:
            return
        from . import utils
        model = self.model
        beta_value = float(model.beta.value())
        xp = np.asarray(self.x_processed.cpu() if isinstance(self.x_processed, torch.Tensor) else self.x_processed)
        xr = np.asarray(self.x_raw.cpu() if isinstance(self.x_raw, torch.Tensor) else self.x_raw)
        offs = np.cumsum([0] + list(model.feature_dimensionalities))
        if self.outdir:
            os.makedirs(self.outdir, exist_ok=True)
        # row selection per feature on the host (visualization.py:17-28), then ONE device call for all features
        picks = [utils.select_display_rows(xr[:, offs[i]:offs[i + 1]], self.max_number_to_display, self.rng)
                 for i in range(model.number_features)]
        n = max(len(inds) for inds, _ in picks)
        row_index = np.stack([np.concatenate([inds, np.full(n - len(inds), inds[-1])]) for inds, _ in picks])
        res = model.compression_matrices(xp, row_index, want=("dist", "comp"))
        comp_all, dist_all = res["comp"].cpu().numpy(), res["dist"].cpu().numpy()
        for i, (inds, sorted_raw) in enumerate(picks):
            k = len(inds)
            rec = dict(epoch=epoch, feature=i, beta=beta_value, compression_matrix=comp_all[i, :k, :k],
                       bhattacharyya=dist_all[i, :k, :k], raw_values=sorted_raw)
            self.matrices.append(rec)
            if self.outdir:
                np.savez(os.path.join(self.outdir, f'feature_{i}_log10beta_{np.log10(beta_value):.3f}.npz'), **rec)


class StashEmbeddingsCallback(Callback):
    """nb-radial cell 5: stash (mu, logvar) of every feature encoder on ``x_in`` every ``save_frequency`` epochs."""

    def __init__(self, save_frequency, x_in, save_start=0):
        super().__init__()
        self.save_frequency = save_frequency
        self.x_in = x_in
        self.mus_for_later = []
        self.logvars_for_later = []
        self.save_start = save_start

    def on_epoch_end(self, epoch, logs=None):
        if (epoch > self.save_start) and ((epoch % self.save_frequency) == 0):
            m = self.model
            E = m.feature_embedding_dimension
            o = m.compression_matrices(self.x_in, None, want=("mu_logvar",))["mu_logvar"].cpu().numpy()
            for i in range(m.number_features):
                self.mus_for_later.append(o[i, :, :E])
                self.logvars_for_later.append(o[i, :, E:])


class InfoPerFeatureCallback(Callback):
    """Callback to compute the information contained in each compression channel during training (models.py:188-223;
    the shipped version passes wrong keyword names to utils -- this follows the corrected copy in nb-radial cell 5).
    ``self.bounds`` collects [lower, upper] (nats) per feature each time it fires, feature-major like the reference."""

    def __init__(self, save_frequency, tf_dataset_validation, evaluation_batch_size=None, number_evaluation_batches=None,
                 info_bound_batch_size=1024, info_bound_number_batches=8, seed=0):
        super().__init__()
        self.save_frequency = save_frequency
        data = tf_dataset_validation[0] if isinstance(tf_dataset_validation, (tuple, list)) else tf_dataset_validation
        self.x_validation = data                                     # the reference maps (x, y) -> x
        self.bounds = []
        self.evaluation_batch_size = evaluation_batch_size or info_bound_batch_size
        self.number_evaluation_batches = number_evaluation_batches or info_bound_number_batches
        self.seed = seed

    def on_epoch_end(self, epoch, logs=None):
        if (epoch % self.save_frequency) != 0:
            return
        from . import utils
        m = self.model
        x = self.x_validation
        xt = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        # all features x all evaluation batches in one grouped encoder pass + one float64 sandwich launch
        lo_up = utils.estimate_mi_sandwich_bounds_all_features(m, xt, evaluation_batch_size=self.evaluation_batch_size,
                                                               number_evaluation_batches=self.number_evaluation_batches,
                                                               seed=self.seed + epoch)
        for i in range(m.number_features):
            self.bounds.append([float(lo_up[i, 0]), float(lo_up[i, 1])])


class ParticleInformationCallback(Callback):
    """nb-particle's information plane and per-particle maps during ``fit`` of a SetTransformerIBNet.  Every
    ``save_frequency`` epochs it appends ``utils.estimate_set_information`` ([lower, upper] nats per set, on
    ``x_validation``: sets as the model takes them) to ``self.bounds``, and with ``probes`` [M, d] also
    ``{epoch, beta, bounds [M, 2]}`` from ``utils.estimate_mi_bounds_at_probes(model.particle_encoder, probes, x_validation)``
    to ``self.probe_bounds``, saved as ``probe_information_log10beta_{log10 beta:.3f}.npz`` under ``outdir`` when given.
    The epoch's draws use ``seed + epoch``.  Neither estimate changes the training run."""

    def __init__(self, save_frequency, x_validation, probes=None, evaluation_batch_size=32, number_evaluation_batches=16,
                 probe_evaluation_batch_size=512, probe_number_evaluation_batches=16, outdir=None, seed=0):
        super().__init__()
        self.save_frequency = save_frequency
        self.x_validation = x_validation
        self.probes = probes
        self.evaluation_batch_size, self.number_evaluation_batches = evaluation_batch_size, number_evaluation_batches
        self.probe_evaluation_batch_size = probe_evaluation_batch_size
        self.probe_number_evaluation_batches = probe_number_evaluation_batches
        self.outdir = outdir
        self.seed = seed
        self.bounds = []
        self.probe_bounds = []

    def on_epoch_end(self, epoch, logs=None):
        if (epoch % self.save_frequency) != 0:
            return
        from . import utils
        m = self.model
        lo_up = utils.estimate_set_information(m, self.x_validation, self.evaluation_batch_size, self.number_evaluation_batches,
                                               seed=self.seed + epoch)
        self.bounds.append([float(lo_up[0]), float(lo_up[1])])
        if self.probes is None:
            return
        beta_value = float(m.beta.value())
        rec = dict(epoch=epoch, beta=beta_value,
                   bounds=utils.estimate_mi_bounds_at_probes(m.particle_encoder, self.probes, self.x_validation,
                                                             self.probe_evaluation_batch_size,
                                                             self.probe_number_evaluation_batches, seed=self.seed + epoch))
        self.probe_bounds.append(rec)
        if self.outdir:
            os.makedirs(self.outdir, exist_ok=True)
            np.savez(os.path.join(self.outdir, f'probe_information_log10beta_{np.log10(beta_value):.3f}.npz'), **rec)


class SimpleEncoder:
    """nb-bool cell 4: "Simple encoder for a binary-valued variable.  With two trainable constants, mu and logvar, this
    encoder maps +1/-1 to a normal distribution with mean +mu/-mu and log variance of logvar."  Stand-alone callable with
    the reference's surface (``mu_scaling``, ``logvar``, ``call``); to TRAIN a bank of them with the fused step build
    ``DistributedIBNet(feature_dimensionalities, 'simple', integration_arch, out, feature_embedding_dimension=1)``."""

    def __init__(self):
        self.mu_scaling = np.ones((1, 1), np.float32)
        self.logvar = -3.0 * np.ones((1, 1), np.float32)

    def build(self, input_shape=None):
        return

    def __call__(self, inputs):
        t = torch.as_tensor(inputs, dtype=torch.float32)
        out = torch.cat([t * float(self.mu_scaling[0, 0]), torch.ones_like(t) * float(self.logvar[0, 0])], -1)
        return _as_numpy_like(inputs, out)

    call = __call__

    @property
    def trainable_variables(self):
        return [self.mu_scaling, self.logvar]


class SharedParticleEncoder:
    """nb-particle cell 8's front end: ONE encoder MLP (positional encoding -> Dense stack -> (mu, logvar)) applied with
    shared weights to every particle of every neighbourhood, logvar offset (-3 there), KL summed over embedding dims AND
    particles and averaged over the batch -- i.e. a one-feature DistributedIBNet on B*particles rows whose KL means are
    taken over B.  The downstream network (the notebook's set transformer) is the caller's: ``encode`` returns
    [B, particles, E] embeddings, ``gradients`` takes d(loss)/d(embeddings) back."""

    def __init__(self, particle_feature_dimensions, particle_encoder_arch_spec, bottleneck_dimension=32,
                 number_positional_encoding_frequencies=5, activation_fn='leaky_relu', leaky_alpha=0.1,
                 logvar_initialization=-3., **kw):
        self.net = DistributedIBNet([int(particle_feature_dimensions)], list(particle_encoder_arch_spec), [], 1,
                                    use_positional_encoding=number_positional_encoding_frequencies > 1,
                                    number_positional_encoding_frequencies=number_positional_encoding_frequencies,
                                    activation_fn=activation_fn, feature_embedding_dimension=bottleneck_dimension,
                                    leaky_alpha=leaky_alpha, logvar_offset=logvar_initialization, **kw)
        self.net.compile(optimizer='adam', loss='external')
        self.beta = self.net.beta
        self.d = int(particle_feature_dimensions)
        self.E = int(bottleneck_dimension)

    def encode(self, batch_inp, eps=None, step=None):
        """batch_inp [B, particles, d] -> (embs_reparam [B, particles, E], kl = mean_B sum_{particles, E})."""
        t = torch.as_tensor(batch_inp, dtype=torch.float32)
        B, Np = t.shape[0], t.shape[1]
        e = None if eps is None else torch.as_tensor(eps, dtype=torch.float32).reshape(B * Np, 1, self.E)
        emb, kl_rows = self.net.encode(t.reshape(B * Np, self.d), eps=e, step=step)
        return emb.reshape(B, Np, self.E), kl_rows[0] * Np

    def gradients(self, batch_inp, d_embs, eps=None, step=None):
        """Flat encoder gradient of (caller's loss + beta * kl) given d(caller's loss)/d(embs_reparam) [B, particles, E]."""
        t = torch.as_tensor(batch_inp, dtype=torch.float32)
        B, Np = t.shape[0], t.shape[1]
        e = None if eps is None else torch.as_tensor(eps, dtype=torch.float32).reshape(B * Np, 1, self.E)
        g, _ = self.net.encoder_gradients(t.reshape(B * Np, self.d), torch.as_tensor(d_embs).reshape(B * Np, self.E),
                                          global_batch=B, eps=e, step=step)
        return g

    def apply_gradients(self, flat_grads):
        self.net.apply_gradients(flat_grads)


def set_transformer_param_specs(d, encoder_arch, E, L, number_heads, key_dim, number_attention_blocks, ff_arch_per_block,
                                final_processing_arch, output_dimensionality, number_positional_encoding_frequencies=5):
    """Every trainable variable of :class:`SetTransformerIBNet` in flat order (nb-particle cell 8's all_trainable_variables):
    a list of (name, shape, init) where init is ('glorot', fan_in, fan_out), 'zeros' or 'ones'.  The attention kernels keep
    their Keras shapes [E, h, dk] / [h, dk, E] here (the flat layout reports them as [E, h*dk] / [h*dk, E]); their glorot
    fans follow Keras' ``_compute_fans`` [KERAS]: fan_in = shape[-2] * prod(shape[:-2]), fan_out = shape[-1] * prod(shape[:-2])."""
    def dense(name, i, o):
        return [(name + "/kernel", (i, o), ("glorot", i, o)), (name + "/bias", (o,), "zeros")]
    specs = []
    width = d * number_positional_encoding_frequencies if number_positional_encoding_frequencies > 1 else d
    dims = [width] + list(encoder_arch) + [2 * E]
    for k in range(len(dims) - 1):
        specs += dense(f"encoder/dense{k}", dims[k], dims[k + 1])
    h, dk = number_heads, key_dim
    for b in range(number_attention_blocks):
        p = f"block{b}/"
        for q in ("query", "key", "value"):
            specs += [(p + q + "/kernel", (E, h, dk), ("glorot", h * E, dk * E)), (p + q + "/bias", (h, dk), "zeros")]
        specs += [(p + "attention_output/kernel", (h, dk, E), ("glorot", dk * h, E * h)), (p + "attention_output/bias", (E,), "zeros")]
        specs += [(p + "ln1/gamma", (E,), "ones"), (p + "ln1/beta", (E,), "zeros")]
        ff = [E] + list(ff_arch_per_block)
        for k in range(len(ff) - 1):
            specs += dense(p + f"ff{k}", ff[k], ff[k + 1])
        specs += [(p + "ln2/gamma", (E,), "ones"), (p + "ln2/beta", (E,), "zeros")]
    head = [E] + list(final_processing_arch) + [output_dimensionality]
    for k in range(len(head) - 1):
        specs += dense(f"head/dense{k}", head[k], head[k + 1])
    return specs


# largest number_particles with variable_set_sizes (include/dib_b200.h: DIB_MAX_VARIABLE_SET_SIZE)
MAX_VARIABLE_SET_SIZE = 256


def check_set_transformer_args(particle_feature_dimensions, particle_encoder_arch_spec, bottleneck_dimension, number_particles,
                               key_dim, number_heads, number_attention_blocks, ff_arch_per_block, ff_activation_fn,
                               final_processing_arch, activation_fn, output_dimensionality, precision, variable_set_sizes=False):
    """The constructor checks of :class:`SetTransformerIBNet` (host only: they run before any device call)."""
    E, L = int(bottleneck_dimension), int(number_particles)
    if int(particle_feature_dimensions) < 1 or int(output_dimensionality) < 1:
        raise ValueError("particle_feature_dimensions and output_dimensionality must be >= 1")
    if any(int(w) < 1 for w in list(particle_encoder_arch_spec) + list(final_processing_arch) + list(ff_arch_per_block)):
        raise ValueError("layer widths must be >= 1")
    if variable_set_sizes and not 1 <= L <= MAX_VARIABLE_SET_SIZE:
        raise ValueError(f"number_particles (the largest set) must be in [1, {MAX_VARIABLE_SET_SIZE}] with variable_set_sizes, "
                         f"got {L}")
    if not variable_set_sizes and not 1 <= L <= 64:
        raise ValueError(f"number_particles must be in [1, 64] (one attention problem per set and head in shared memory; up to "
                         f"{MAX_VARIABLE_SET_SIZE} with variable_set_sizes=True), got {L}")
    if not 1 <= int(key_dim) <= 128 or int(number_heads) < 1 or int(number_attention_blocks) < 1:
        raise ValueError("the attention needs key_dim in [1, 128], number_heads >= 1 and number_attention_blocks >= 1")
    if (int(number_heads) * int(key_dim)) % 4 or E % 4 or E > 128:
        raise ValueError("number_heads * key_dim and bottleneck_dimension must be multiples of 4, bottleneck_dimension <= 128")
    if not ff_arch_per_block or int(ff_arch_per_block[-1]) != E:
        raise ValueError(f"the last width of ff_arch_per_block must equal bottleneck_dimension ({E}): the block adds FF(H) to H")
    for a in (ff_activation_fn, activation_fn):
        if a not in _lib.ACTIVATIONS:
            raise ValueError(f"unsupported activation {a!r}")
    if precision not in _lib.PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(_lib.PRECISIONS)}, got {precision!r}")


def pad_sets(sets, max_set_size):
    """Sets of different sizes -- a list of N arrays [l_i, d], e.g. nb-particle's neighbourhoods before ``np.stack`` -- as
    (x [N, max_set_size, d] float32 with zero padding rows, set_sizes [N] int32), the pair a variable-size
    :class:`SetTransformerIBNet` takes."""
    arrs = [np.asarray(a, dtype=np.float32) for a in sets]
    if not arrs:
        raise ValueError("pad_sets needs at least one set")
    L = int(max_set_size)
    d = arrs[0].shape[-1] if arrs[0].ndim == 2 else -1
    for i, a in enumerate(arrs):
        if a.ndim != 2 or a.shape[1] != d:
            raise ValueError(f"set {i} has shape {a.shape}; every set must be [particles, {d}]")
    sizes = np.array([a.shape[0] for a in arrs], dtype=np.int32)
    check_set_sizes(sizes, len(arrs), L)
    x = np.zeros((len(arrs), L, d), dtype=np.float32)
    for i, a in enumerate(arrs):
        x[i, :a.shape[0]] = a
    return x, sizes


def check_set_sizes(sizes, n, max_set_size):
    """Host check of the sizes of n padded sets: an int array [n] with 1 <= size <= max_set_size."""
    s = np.asarray(sizes)
    if s.shape != (int(n),):
        raise ValueError(f"set_sizes has shape {s.shape}; expected one size per set, ({int(n)},)")
    if s.size and (s.min() < 1 or s.max() > int(max_set_size)):
        bad = s[(s < 1) | (s > int(max_set_size))][0]
        raise ValueError(f"set sizes must be in [1, {int(max_set_size)}], got {int(bad)}")


class _ParticleEncoder(_FeatureEncoder):
    """model.particle_encoder: [..., d] -> [..., 2E] = (mu || logvar), logvar offset applied (dib_encode_feature on particle
    rows).  ``utils.estimate_mi_sandwich_bounds(model.particle_encoder, particles [N, d])`` works on it.  A variable-size model
    also takes a list of [l_i, d] sets (-> a list of [l_i, 2E]) or a pair (x [N, Lmax, d], set_sizes [N]) (-> [N, Lmax, 2E],
    padding rows zero); only the real particles are encoded."""

    def __call__(self, x, training=None):
        m = self._model
        if m.variable_set_sizes and isinstance(x, (list, tuple)):
            if isinstance(x, list):
                rows = np.concatenate([np.asarray(a, dtype=np.float32).reshape(-1, m.particle_feature_dimensions) for a in x])
                out = m._encode_feature(0, torch.from_numpy(rows)).cpu().numpy()
                return np.split(out, np.cumsum([len(a) for a in x])[:-1])
            xd, sd = m._inputs(x)
            L = m.number_particles
            real = (torch.arange(L, device=m.device)[None, :] < sd[:, None].long()).reshape(-1)
            out = torch.zeros(xd.shape[0] * L, 2 * m.feature_embedding_dimension, dtype=torch.float32, device=m.device)
            out[real] = m._encode_feature(0, xd.reshape(-1, m.particle_feature_dimensions)[real])
            return _as_numpy_like(x[0], out.reshape(xd.shape[0], L, -1))
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        out = m._encode_feature(0, t)
        return _as_numpy_like(x, out.reshape(*t.shape[:-1], out.shape[-1]))


class SetTransformerIBNet(DistributedIBNet):
    """nb-particle cell 8 (BASELINE config 5): a shared particle encoder (positional encoding -> Dense stack -> (mu, logvar),
    logvar + ``logvar_initialization``, reparameterised per particle) feeding a set transformer -- ``number_attention_blocks``
    blocks of ``H = LayerNorm(x + MultiHeadAttention(number_heads, key_dim)(x, x, x))``, ``x = LayerNorm(H + FF(H))`` --, the
    mean over the particles and a Dense head.  Loss = compiled loss + beta * KL, the KL summed over dims and particles and
    averaged over sets.  The whole step runs in the library (dib_config.integration_kind = set transformer), so ``compile`` /
    ``fit`` / ``train_on_batch`` / ``evaluate`` / ``predict``, CUDA-graph replay and the data-parallel all-reduce are the
    ones of :class:`DistributedIBNet`.

    ``x`` is [N, number_particles, particle_feature_dimensions] and ``y`` [N, output_dimensionality]; batches count sets.
    ``model.particle_encoder(x)`` returns mu || logvar per particle and ``model.set_transformer(embs)`` runs the network
    after the encoder.  History keys: loss, accuracy (with metrics=['accuracy']), KL0 (per set), beta and their val_ twins.
    ``fp16`` / ``bf16`` run every dense layer on the TF32 kernels; the attention and LayerNorm kernels are fp32 in every mode.

    ``variable_set_sizes=True`` takes sets of different sizes, up to ``number_particles`` (at most 256) particles each -- the
    notebook's ragged neighbourhoods without clipping them to one size.  Wherever ``x`` goes (``fit`` and its
    ``validation_data``, ``evaluate``, ``predict``, ``train_on_batch``, ``compute_gradients``, calling the model), pass either a
    list of N arrays [l_i, d] or a pair (x_padded [N, number_particles, d], set_sizes [N]) (see :func:`pad_sets`).  Each set's
    loss, KL, prediction and gradient are the fixed-size model's with number_particles = l_i on its real particles: padding keys
    are masked out of the attention (Keras' attention_mask), the mean runs over the real particles, the KL sums over them, and
    what the padding rows hold is ignored.  ``model.set_transformer(embs, set_sizes=...)`` takes the sizes of padded
    embeddings [N, number_particles, E] (or a list of [l_i, E])."""

    def __init__(self, particle_feature_dimensions, particle_encoder_arch_spec, bottleneck_dimension=32, number_particles=50,
                 key_dim=128, number_heads=12, number_attention_blocks=6, ff_arch_per_block=None, ff_activation_fn='relu',
                 final_processing_arch=(256,), activation_fn='leaky_relu', leaky_alpha=0.1, output_dimensionality=1,
                 logvar_initialization=-3., number_positional_encoding_frequencies=5, precision='fp32', variable_set_sizes=False,
                 **kw):
        E = int(bottleneck_dimension)
        ff = [128, E] if ff_arch_per_block is None else [int(w) for w in ff_arch_per_block]
        check_set_transformer_args(particle_feature_dimensions, particle_encoder_arch_spec, E, number_particles, key_dim,
                                   number_heads, number_attention_blocks, ff, ff_activation_fn, final_processing_arch,
                                   activation_fn, output_dimensionality, precision, bool(variable_set_sizes))
        self.variable_set_sizes = bool(variable_set_sizes)
        self.particle_feature_dimensions = int(particle_feature_dimensions)
        self.number_particles = int(number_particles)
        self.key_dim, self.number_heads = int(key_dim), int(number_heads)
        self.number_attention_blocks = int(number_attention_blocks)
        self.ff_arch_per_block, self.ff_activation_fn = ff, ff_activation_fn
        self.final_processing_arch = [int(w) for w in final_processing_arch]
        # the host sees one row of number_particles * d values per set; the library runs the encoder on the particle rows
        super().__init__([self.number_particles * self.particle_feature_dimensions], list(particle_encoder_arch_spec),
                         self.final_processing_arch, output_dimensionality,
                         use_positional_encoding=number_positional_encoding_frequencies > 1,
                         number_positional_encoding_frequencies=number_positional_encoding_frequencies,
                         activation_fn=activation_fn, feature_embedding_dimension=E, output_activation_fn=None,
                         precision=precision, leaky_alpha=leaky_alpha, logvar_offset=logvar_initialization, **kw)
        n_enc = 2 * (len(self.feature_encoder_architecture) + 1)
        self.particle_encoder = _ParticleEncoder(self, 0, range(n_enc))
        self.feature_encoders = [self.particle_encoder]
        # embeddings [n, L, E] -> [n, out] through the attention blocks, the mean over the particles and the head
        self.set_transformer = _IntegrationNetwork(self, range(n_enc, self._n_model_vars), self.number_particles * E)
        self.integration_network = self.set_transformer

    def _config(self, max_batch):
        cfg = super()._config(max_batch)
        self._c_pd = (ctypes.c_int32 * 1)(self.particle_feature_dimensions)
        self._c_ff = (ctypes.c_int32 * len(self.ff_arch_per_block))(*self.ff_arch_per_block)
        cfg.feature_dimensionalities = self._c_pd
        cfg.integration_kind = _lib.INTEGRATION_KINDS["set_transformer"]
        cfg.set_size = self.number_particles
        cfg.number_attention_blocks = self.number_attention_blocks
        cfg.number_heads, cfg.key_dim = self.number_heads, self.key_dim
        cfg.number_ff_layers, cfg.ff_architecture = len(self.ff_arch_per_block), self._c_ff
        cfg.ff_activation_fn = _lib.ACTIVATIONS[self.ff_activation_fn]
        cfg.layer_norm_epsilon = 1e-3                                        # [KERAS] LayerNormalization default
        cfg.variable_set_sizes = int(self.variable_set_sizes)
        return cfg

    def _device_sizes(self, sizes, n):
        """Set sizes checked on the host (one read of a device tensor), then as int32 on the device."""
        host = sizes.detach().cpu().numpy() if isinstance(sizes, torch.Tensor) else np.asarray(sizes)
        if host.dtype.kind not in "iu":
            raise ValueError(f"set_sizes must be integers, got {host.dtype}")
        check_set_sizes(host, n, self.number_particles)
        if isinstance(sizes, torch.Tensor):
            return sizes.to(device=self.device, dtype=torch.int32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(host, dtype=np.int32)).to(self.device)

    def _inputs(self, x):
        """Variable set sizes: a list of [l_i, d] sets or a pair (x [N, Lmax, d], set_sizes [N]) -> (x [N, Lmax * d] on the
        device, int32 sizes on the device), the sizes checked before any device work."""
        if not self.variable_set_sizes:
            return super()._inputs(x)
        L, d = self.number_particles, self.particle_feature_dimensions
        if isinstance(x, list):
            x = pad_sets(x, L)
        if not (isinstance(x, tuple) and len(x) == 2):
            raise ValueError("a SetTransformerIBNet with variable_set_sizes takes a list of [particles, d] arrays or a pair "
                             "(x_padded [N, number_particles, d], set_sizes [N])")
        xp, sizes = x
        shape = tuple(xp.shape)
        if len(shape) != 3 or shape[1:] != (L, d):
            raise ValueError(f"padded x has shape {shape}; expected [N, {L}, {d}]")
        sd = self._device_sizes(sizes, shape[0])
        return self._to_device(xp, L * d), sd

    def _integration_inputs(self, emb, set_sizes, width):
        if not self.variable_set_sizes:
            return super()._integration_inputs(emb, set_sizes, width)
        E = self.feature_embedding_dimension
        if isinstance(emb, list):
            if set_sizes is not None:
                raise ValueError("a list of embeddings carries its own set sizes")
            emb, set_sizes = pad_sets(emb, self.number_particles)
        if set_sizes is None:
            raise ValueError("model.set_transformer of a variable-size model needs set_sizes (or a list of [l_i, E] embeddings)")
        if len(emb.shape) != 3 or tuple(emb.shape[1:]) != (self.number_particles, E):
            raise ValueError(f"embeddings have shape {tuple(emb.shape)}; expected [N, {self.number_particles}, {E}]")
        sd = self._device_sizes(set_sizes, emb.shape[0])
        return self._to_device(emb, width), sd

    def predict(self, x, batch_size=32, **_):
        if not self.variable_set_sizes:
            return super().predict(x, batch_size)
        if isinstance(x, list):
            x = pad_sets(x, self.number_particles)
        xp, sizes = x
        self._device_sizes(sizes, xp.shape[0])                  # checked once, before any device work
        outs, n = [], xp.shape[0]
        st = self._inference_step()
        for b0 in range(0, n, int(batch_size)):
            o = self((xp[b0:b0 + int(batch_size)], sizes[b0:b0 + int(batch_size)]), training=False, step=st, sample_offset=b0)
            outs.append(o if isinstance(xp, torch.Tensor) else np.asarray(o))
        return torch.cat(outs) if isinstance(xp, torch.Tensor) else np.concatenate(outs)

    def param_specs(self):
        """(name, Keras shape, init) of every trainable variable in flat order; see :func:`set_transformer_param_specs`."""
        return set_transformer_param_specs(self.particle_feature_dimensions, self.feature_encoder_architecture,
                                           self.feature_embedding_dimension, self.number_particles, self.number_heads,
                                           self.key_dim, self.number_attention_blocks, self.ff_arch_per_block,
                                           self.final_processing_arch, self.output_dimensionality,
                                           self.number_positional_encoding_frequencies if self.use_positional_encoding else 1)

    def _param_inits(self):
        """[KERAS] glorot_uniform kernels with the fans of ``_compute_fans`` (3-D attention kernels included), zero biases,
        LayerNorm gamma = 1 and beta = 0."""
        return [init for _, _, init in self.param_specs()]

    def _encoder_rows(self, i, x_i):
        """Particle rows [..., d] -> [rows, d]; the handle is sized in sets of number_particles rows."""
        t = self._to_device(x_i).reshape(-1, self.particle_feature_dimensions).contiguous()
        return t, max(1, -(-t.shape[0] // self.number_particles))

    def compile(self, optimizer='adam', loss=None, metrics=None, **kw):
        kind = resolve_loss(loss)
        if kind in ("sparse_ce_logits", "infonce"):
            raise ValueError("SetTransformerIBNet trains with BinaryCrossentropy (logits or probabilities), MSE or the external "
                             f"loss, not {kind!r}")
        super().compile(optimizer, loss, metrics, **kw)

    def build(self, input_shape):
        assert tuple(input_shape[-2:]) == (self.number_particles, self.particle_feature_dimensions)

    def compression_matrices(self, *a, **k):
        raise NotImplementedError("compression matrices of particles: run model.particle_encoder on the particle rows and "
                                  "utils.bhattacharyya_dist_mat on its output")
