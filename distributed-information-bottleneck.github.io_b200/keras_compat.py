"""The slice of the tf.keras surface that the reference's training driver touches (train.py:128-172,
nb-radial cell 10): optimizer/loss objects handed to ``model.compile``, the ``Callback`` protocol and ``History``.
These are thin descriptions -- the arithmetic they name runs in the CUDA library."""
from __future__ import annotations


class Adam:
    """tf.keras.optimizers.Adam(learning_rate, beta_1, beta_2, epsilon) -- Keras defaults; epsilon is applied
    outside the bias correction (dib_adam_step)."""

    def __init__(self, learning_rate=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-7, name="adam"):
        self.learning_rate = learning_rate
        self.beta_1, self.beta_2, self.epsilon = beta_1, beta_2, epsilon
        self.name = name

    lr = property(lambda self: self.learning_rate, lambda self, v: setattr(self, "learning_rate", v))


class SGD:
    """tf.keras.optimizers.SGD(learning_rate=0.01, momentum=0.0, nesterov=False):
    v = momentum * v - lr * g;  w += momentum * v - lr * g if nesterov else v   (dib_optimizer_step kind 0)."""
    kind = 0

    def __init__(self, learning_rate=0.01, momentum=0.0, nesterov=False, name="SGD"):
        self.learning_rate, self.momentum, self.nesterov, self.name = learning_rate, float(momentum), bool(nesterov), name

    lr = property(lambda self: self.learning_rate, lambda self, v: setattr(self, "learning_rate", v))

    def hyper(self):
        return self.momentum, 1.0 if self.nesterov else 0.0, 0.0


class RMSprop:
    """tf.keras.optimizers.RMSprop(learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-7) (non-centered), TensorFlow's
    ApplyRMSProp: ms = rho ms + (1-rho) g^2;  mom = momentum mom + lr g / sqrt(ms + eps);  w -= mom  (kind 1)."""
    kind = 1

    def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-7, centered=False, name="RMSprop"):
        if centered:
            raise NotImplementedError("RMSprop(centered=True) is not implemented")
        self.learning_rate, self.rho, self.momentum, self.epsilon, self.name = learning_rate, float(rho), float(momentum), float(epsilon), name

    lr = property(lambda self: self.learning_rate, lambda self, v: setattr(self, "learning_rate", v))

    def hyper(self):
        return self.rho, self.momentum, self.epsilon


class optimizers:
    Adam = Adam
    SGD = SGD
    RMSprop = RMSprop

    @staticmethod
    def get(identifier):
        """tf.keras.optimizers.get(name) as used at train.py:128 (the --optimizer flag, train.py:41)."""
        if isinstance(identifier, (Adam, SGD, RMSprop)):
            return identifier
        if isinstance(identifier, str):
            table = {"adam": Adam, "sgd": SGD, "rmsprop": RMSprop}
            if identifier.lower() in table:
                return table[identifier.lower()]()
        raise ValueError(f"optimizer {identifier!r} is not implemented by the engine (adam, sgd, rmsprop are)")


class _Loss:
    kind = None

    def __init__(self, from_logits=False, name=None):
        self.from_logits = from_logits
        self.name = name


class BinaryCrossentropy(_Loss):
    """data.py:65 / nb-radial: BinaryCrossentropy(from_logits=True); from_logits=False (the Keras default) is the
    clipped-probability form for models with output_activation_fn='sigmoid'."""
    kind = "bce_logits"
    kind_probs = "bce_probs"


class SparseCategoricalCrossentropy(_Loss):
    """data.py:343: SparseCategoricalCrossentropy(from_logits=True)."""
    kind = "sparse_ce_logits"


class MeanSquaredError(_Loss):
    kind = "mse"

    def __init__(self, name=None):
        super().__init__(from_logits=True, name=name)


class InfoNCE(_Loss):
    """The InfoNCE path of train.py:180-289 (``--infonce_loss``; the double pendulum's loss, data.py:131) as a compiled loss.

    The model is trained together with an output encoder for y -- positional encoding as the model's, ``Dense(h,
    activation_fn)`` for every width of ``y_encoder_architecture``, then a linear ``Dense(output_dimensionality)``
    (train.py:186-193) -- on the symmetric InfoNCE of train.py:201-213 between ``model(x)`` and ``output_encoder(y)``:
    ``mean_i CE(i, S[i,:]) + mean_i CE(i, S^T[i,:])`` with ``S = get_scaled_similarity(., ., similarity, temperature)``.
    Defaults are train.py:55-62's.  ``y_dimensionality`` is the width of y (it sizes the output encoder).

    ``negatives`` says which rows are the negatives of a row when the model is data parallel, because that choice changes
    the loss.  ``'global'``: all other rows of the global batch, so N processes compute exactly the one-process loss of that
    batch (DESIGN.md section 7).  ``None`` (default): no choice made; one process trains as always, and a process group of
    more than one rank is refused."""
    kind = "infonce"

    def __init__(self, y_dimensionality, y_encoder_architecture=(128, 128), similarity="l2", temperature=1.0, name=None,
                 negatives=None):
        from .utils import SIMILARITY_TYPES
        super().__init__(from_logits=True, name=name)
        if negatives not in (None, "global"):
            raise ValueError(f"negatives must be None or 'global', got {negatives!r}")
        self.negatives = negatives
        if similarity not in SIMILARITY_TYPES:
            raise ValueError(f"similarity must be one of {sorted(SIMILARITY_TYPES)}, got {similarity!r}")
        if not float(temperature) > 0:
            raise ValueError("temperature must be > 0")
        self.y_dimensionality = int(y_dimensionality)
        self.y_encoder_architecture = [int(h) for h in y_encoder_architecture]
        if self.y_dimensionality < 1 or any(h < 1 for h in self.y_encoder_architecture):
            raise ValueError("y_dimensionality and the output-encoder widths must be >= 1")
        self.similarity = similarity
        self.temperature = float(temperature)

    def spec(self):
        """What shapes the handle: equal specs share the output encoder's layout and kernels."""
        return (self.y_dimensionality, tuple(self.y_encoder_architecture), self.similarity, self.temperature)


class losses:
    BinaryCrossentropy = BinaryCrossentropy
    SparseCategoricalCrossentropy = SparseCategoricalCrossentropy
    MeanSquaredError = MeanSquaredError
    InfoNCE = InfoNCE


def resolve_loss(loss):
    if isinstance(loss, _Loss):
        if not loss.from_logits:
            if getattr(loss, "kind_probs", None):
                return loss.kind_probs
            raise NotImplementedError(
                f"{type(loss).__name__}(from_logits=False) is not implemented: the reference's call sites pass logits")
        return loss.kind
    if isinstance(loss, str):
        key = loss.lower()
        if key in ("mse", "mean_squared_error"):
            return "mse"
        if key in ("bce_logits", "sparse_ce_logits", "bce_probs"):
            return key
        if key == "binary_crossentropy":               # the Keras string means from_logits=False
            return "bce_probs"
        if key in ("external", "custom"):       # GradientTape-style loops: the caller owns the task loss
            return "external"
        if key == "infonce":                    # what data.py:131 returns for the pendulum
            raise ValueError("loss='infonce' needs the width of y and the output-encoder architecture: "
                             "compile with loss=losses.InfoNCE(y_dimensionality=..., y_encoder_architecture=[...])")
    raise ValueError(f"unsupported loss {loss!r}")


from .metrics import metrics  # noqa: E402,F401 -- keras.metrics: the compiled metrics' objects


class Callback:
    """tf.keras.callbacks.Callback protocol (models.py:125,152,188): the trainer sets ``.model``."""
    model = None

    def set_model(self, model):
        self.model = model

    def on_train_begin(self, logs=None): pass
    def on_train_end(self, logs=None): pass
    def on_epoch_begin(self, epoch, logs=None): pass
    def on_epoch_end(self, epoch, logs=None): pass
    def on_train_batch_begin(self, batch, logs=None): pass
    def on_train_batch_end(self, batch, logs=None): pass


class callbacks:
    Callback = Callback


class History(Callback):
    """Return value of Model.fit: ``.history`` maps metric name -> list over epochs (train.py:169-172)."""

    def __init__(self):
        self.history = {}
        self.epoch = []

    def on_epoch_end(self, epoch, logs=None):
        self.epoch.append(epoch)
        for k, v in (logs or {}).items():
            self.history.setdefault(k, []).append(v)
