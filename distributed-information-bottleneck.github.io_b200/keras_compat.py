"""The slice of the tf.keras surface that the reference's training driver touches (train.py:128-172,
nb-radial cell 10): optimizer/loss objects handed to ``model.compile``, the ``Callback`` protocol and ``History``.
These are thin descriptions -- the arithmetic they name runs in the CUDA library."""
from __future__ import annotations

import os
import warnings

import numpy as np


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


class History(Callback):
    """Return value of Model.fit: ``.history`` maps metric name -> list over epochs (train.py:169-172)."""

    def __init__(self):
        self.history = {}
        self.epoch = []

    def on_epoch_end(self, epoch, logs=None):
        self.epoch.append(epoch)
        for k, v in (logs or {}).items():
            self.history.setdefault(k, []).append(v)


def _higher_is_better(monitor):
    """mode='auto': accuracy-, AUC-, precision- and recall-like names are maximised, everything else minimised."""
    name = monitor.removeprefix("val_")
    return "acc" in name or "auc" in name or "precision" in name or "recall" in name or name.startswith("fmeasure")


class ModelCheckpoint(Callback):
    """tf.keras.callbacks.ModelCheckpoint (Keras 2): at every epoch end, save the model (``model.save``) or its weights
    (``save_weights_only``) to ``filepath.format(epoch=epoch + 1, **logs)``.  With ``save_best_only`` the file is written
    only when ``logs[monitor]`` improves on the best value so far (``initial_value_threshold`` is the starting best); an
    epoch whose logs lack ``monitor`` is skipped with a warning.  ``mode`` is 'min', 'max' or 'auto' ('max' for accuracy /
    AUC / precision / recall names).  Only ``save_freq='epoch'`` is implemented."""

    def __init__(self, filepath, monitor="val_loss", verbose=0, save_best_only=False, save_weights_only=False, mode="auto",
                 save_freq="epoch", options=None, initial_value_threshold=None):
        super().__init__()
        if save_freq != "epoch":
            if isinstance(save_freq, int) and not isinstance(save_freq, bool):
                raise ValueError(f"ModelCheckpoint(save_freq={save_freq}): saving every so many batches is not implemented; "
                                 "use save_freq='epoch'")
            raise ValueError(f"Unrecognized save_freq: {save_freq!r}")
        if options is not None:
            raise ValueError("ModelCheckpoint(options=...) is not implemented")
        self.filepath = os.fspath(filepath)
        self.monitor = monitor
        self.verbose = verbose
        self.save_best_only = bool(save_best_only)
        self.save_weights_only = bool(save_weights_only)
        self.save_freq = save_freq
        if mode not in ("auto", "min", "max"):
            warnings.warn(f"ModelCheckpoint mode {mode!r} is unknown, fallback to auto mode.")
            mode = "auto"
        self.mode = mode
        self._maximize = mode == "max" or (mode == "auto" and _higher_is_better(monitor))
        self.best = (float(initial_value_threshold) if initial_value_threshold is not None
                     else (-np.inf if self._maximize else np.inf))

    def _improved(self, current):
        return current > self.best if self._maximize else current < self.best

    def on_epoch_end(self, epoch, logs=None):
        logs = logs or {}
        path = self.filepath.format(epoch=epoch + 1, **logs)
        if self.save_best_only:
            current = logs.get(self.monitor)
            if current is None:
                warnings.warn(f"Can save best model only with {self.monitor} available, skipping.")
                return
            if not self._improved(current):
                if self.verbose:
                    print(f"\nEpoch {epoch + 1}: {self.monitor} did not improve from {self.best:.5f}")
                return
            if self.verbose:
                print(f"\nEpoch {epoch + 1}: {self.monitor} improved from {self.best:.5f} to {current:.5f}, saving to {path}")
            self.best = current
        elif self.verbose:
            print(f"\nEpoch {epoch + 1}: saving model to {path}")
        if self.save_weights_only:
            self.model.save_weights(path)
        else:
            self.model.save(path)


class BackupAndRestore(Callback):
    """tf.keras.callbacks.BackupAndRestore: the full training state (``model.save``) goes to ``backup_dir`` at every epoch
    end.  ``on_train_begin`` restores it when a backup exists and makes ``fit`` continue with the epoch after the last
    completed one, so a run killed between epochs and started again with the same ``fit`` call ends where the uninterrupted
    run ends -- bit for bit, as every random draw is keyed by saved state.  ``on_train_end`` deletes the backup when
    ``delete_checkpoint``; an exception that escapes ``fit`` skips it, so the backup survives."""

    FILENAME = "backup.npz"

    def __init__(self, backup_dir, save_freq="epoch", delete_checkpoint=True):
        super().__init__()
        if save_freq != "epoch":
            raise ValueError(f"BackupAndRestore(save_freq={save_freq!r}): only backups at epoch ends are implemented")
        if not backup_dir:
            raise ValueError("BackupAndRestore needs a backup_dir")
        self.backup_dir = os.fspath(backup_dir)
        self.delete_checkpoint = bool(delete_checkpoint)
        self.path = os.path.join(self.backup_dir, self.FILENAME)

    def on_train_begin(self, logs=None):
        epochs_done = self.model._restore_backup(self.path)
        if epochs_done is not None:
            self.model._resume_epoch = epochs_done

    def on_epoch_end(self, epoch, logs=None):
        if self.model._is_writer():
            os.makedirs(self.backup_dir, exist_ok=True)
        self.model.save(self.path)

    def on_train_end(self, logs=None):
        if self.delete_checkpoint and self.model._is_writer():
            try:
                os.remove(self.path)
                os.rmdir(self.backup_dir)
            except OSError:                    # already gone, or the directory holds other files
                pass



class callbacks:
    Callback = Callback
    History = History
    ModelCheckpoint = ModelCheckpoint
    BackupAndRestore = BackupAndRestore
