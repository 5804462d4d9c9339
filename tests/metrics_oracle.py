"""Float64 restatement of the Keras 2 metrics that ``compile(metrics=, weighted_metrics=)`` computes on the device.

Every item marked [KERAS] restates what tf.keras 2.x does (keras/metrics, keras/losses, keras/backend and
keras/utils/metrics_utils); the tests pin these classes against scikit-learn and against closed forms, and then the
library's metric tail against them.  Rows are the model's outputs z [n, out], targets y ([n, out], or [n] class labels for
the sparse metrics) and sample weights w [n] (None: 1).
"""
import numpy as np

EPSILON = 1e-7                     # [KERAS] keras.backend.epsilon()
# [KERAS] backend.binary_crossentropy / sparse_categorical_crossentropy clip to [epsilon_, 1 - epsilon_] with epsilon_ a float32
# constant, so the upper bound is the float32 1 - 2^-23, not 1 - 1e-7: 1 - p + eps is then 2.19e-7 at the clip, not 2e-7
CLIP_LO = float(np.float32(EPSILON))
CLIP_HI = float(np.float32(1.0) - np.float32(EPSILON))


def sigmoid(z):
    z = np.asarray(z, np.float64)
    return np.where(z >= 0, 1.0 / (1.0 + np.exp(-np.abs(z))), np.exp(-np.abs(z)) / (1.0 + np.exp(-np.abs(z))))


def _rows(z, y, cols):
    z = np.asarray(z, np.float64)
    z = z.reshape(len(z), -1)
    y = np.asarray(y, np.float64)
    return z, (y.reshape(len(z), -1) if cols else y.reshape(len(z)))


# ---------------------------------------------------------------------------------------------------------------------
# per-row values of the mean metrics (MeanMetricWrapper functions; each reduces the last axis by its mean)
# ---------------------------------------------------------------------------------------------------------------------
def mse_rows(z, y):
    """[KERAS] keras.losses.mean_squared_error: mean(square(y_pred - y_true), axis=-1)."""
    z, y = _rows(z, y, True)
    return np.mean((z - y) ** 2, axis=-1)


def mae_rows(z, y):
    """[KERAS] keras.losses.mean_absolute_error: mean(abs(y_pred - y_true), axis=-1)."""
    z, y = _rows(z, y, True)
    return np.mean(np.abs(z - y), axis=-1)


def binary_accuracy_rows(z, y, threshold=0.5):
    """[KERAS] keras.metrics.binary_accuracy: mean(equal(y_true, cast(y_pred > threshold)), axis=-1)."""
    z, y = _rows(z, y, True)
    return np.mean((y == (z > threshold).astype(np.float64)).astype(np.float64), axis=-1)


def sparse_categorical_accuracy_rows(z, y):
    """[KERAS] keras.metrics.sparse_categorical_accuracy: equal(y_true, cast(argmax(y_pred, -1), floatx)) (first maximum)."""
    z, y = _rows(z, y, False)
    return (y == np.argmax(z, axis=-1).astype(np.float64)).astype(np.float64)


def binary_crossentropy_rows(z, y, from_logits=False):
    """[KERAS] keras.losses.binary_crossentropy -> keras.backend.binary_crossentropy, mean over axis -1.  from_logits:
    tf.nn.sigmoid_cross_entropy_with_logits = max(z, 0) - z y + log(1 + exp(-|z|)).  Otherwise the probabilities are
    clipped to [eps, 1 - eps] (float32 bounds: CLIP_LO, CLIP_HI) and bce = -(y log(p + eps) + (1 - y) log(1 - p + eps)); the
    string 'binary_crossentropy' is this form whatever the model outputs."""
    z, y = _rows(z, y, True)
    if from_logits:
        v = np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z)))
    else:
        p = np.clip(z, CLIP_LO, CLIP_HI)
        v = -(y * np.log(p + CLIP_LO) + (1 - y) * np.log(1 - p + CLIP_LO))
    return np.mean(v, axis=-1)


def sparse_categorical_crossentropy_rows(z, y, from_logits=False):
    """[KERAS] keras.backend.sparse_categorical_crossentropy: targets cast to int64; from_logits=False clips the outputs to
    [eps, 1 - eps] and takes their log, then tf.nn.sparse_softmax_cross_entropy_with_logits: -log_softmax(o)[label], i.e.
    -log(p~_label / sum_j p~_j) on probabilities.  A label outside [0, C) gives NaN (TensorFlow on a GPU)."""
    z, y = _rows(z, y, False)
    o = z if from_logits else np.log(np.clip(z, CLIP_LO, CLIP_HI))
    m = o.max(axis=-1, keepdims=True)
    lse = (m + np.log(np.exp(o - m).sum(axis=-1, keepdims=True)))[:, 0]
    ok = np.isfinite(y) & (y > -1) & (y < z.shape[1])
    lab = np.where(ok, np.trunc(np.where(ok, y, 0)), 0).astype(np.int64)
    return np.where(ok, lse - o[np.arange(len(z)), lab], np.nan)


ROW_FUNCTIONS = {
    "mse": lambda z, y, m: mse_rows(z, y),
    "mae": lambda z, y, m: mae_rows(z, y),
    "binary_accuracy": lambda z, y, m: binary_accuracy_rows(z, y, m.get("threshold", 0.5)),
    "sparse_categorical_accuracy": lambda z, y, m: sparse_categorical_accuracy_rows(z, y),
    "binary_crossentropy": lambda z, y, m: binary_crossentropy_rows(z, y, m.get("from_logits", False)),
    "sparse_categorical_crossentropy": lambda z, y, m: sparse_categorical_crossentropy_rows(z, y, m.get("from_logits", False)),
}


class Mean:
    """[KERAS] keras.metrics.Mean (Reduction.WEIGHTED_MEAN), stateful over update_state calls: total += sum w v,
    count += sum w; result = divide_no_nan(total, count).  Keras keeps float32 variables; this keeps float64."""

    def __init__(self, kind, **params):
        self.kind, self.params = kind, params
        self.total = self.count = 0.0

    def update(self, z, y, w=None):
        v = ROW_FUNCTIONS[self.kind](z, y, self.params)
        w = np.ones(len(v)) if w is None else np.asarray(w, np.float64).reshape(-1)
        self.total += float(np.sum(w * v))
        self.count += float(np.sum(w))

    def result(self):
        return self.total / self.count if self.count != 0 else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# confusion-matrix metrics (one output)
# ---------------------------------------------------------------------------------------------------------------------
def auc_thresholds(num_thresholds):
    """[KERAS] keras.metrics.AUC.__init__: [0 - epsilon] + [(i + 1) / (T - 1) for i in range(T - 2)] + [1 + epsilon], held
    as a float32 constant (so the comparison p > t is against the float32 value)."""
    T = int(num_thresholds)
    t = [0.0 - EPSILON] + [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)] + [1.0 + EPSILON]
    return np.asarray(t, np.float32).astype(np.float64)


def confusion(p, y, w, thresholds):
    """[KERAS] metrics_utils.update_confusion_matrix_variables: y_true cast to bool (positive when != 0), a prediction is
    positive at t when p > t (strict); TP, FP, TN, FN [T] are the summed sample weights (1 each without weights)."""
    p = np.asarray(p, np.float64).reshape(-1)
    pos = np.asarray(y, np.float64).reshape(-1) != 0
    w = np.ones(len(p)) if w is None else np.asarray(w, np.float64).reshape(-1)
    above = p[None, :] > np.asarray(thresholds, np.float64)[:, None]          # [T, n]; NaN exceeds nothing
    tp = (above & pos).astype(np.float64) @ w
    fp = (above & ~pos).astype(np.float64) @ w
    fn = (~above & pos).astype(np.float64) @ w
    tn = (~above & ~pos).astype(np.float64) @ w
    return tp, fp, tn, fn


def _div(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.divide(a, b, out=np.zeros(np.broadcast(a, b).shape), where=b != 0)       # [KERAS] tf.math.divide_no_nan


class AUC:
    """[KERAS] keras.metrics.AUC (multi_label=False): from_logits applies sigmoid first; result() integrates the ROC or PR
    curve over the thresholds with the interpolation (trapezoids; PR: interpolate_pr_auc, Davis & Goadrich 2006),
    minoring or majoring Riemann sums."""

    def __init__(self, num_thresholds=200, curve="ROC", summation_method="interpolation", from_logits=False):
        self.thresholds = auc_thresholds(num_thresholds)
        self.curve, self.summation_method, self.from_logits = curve, summation_method, from_logits
        T = len(self.thresholds)
        self.tp, self.fp, self.tn, self.fn = (np.zeros(T) for _ in range(4))

    def update(self, z, y, w=None):
        p = sigmoid(z) if self.from_logits else np.asarray(z, np.float64)
        for acc, v in zip((self.tp, self.fp, self.tn, self.fn), confusion(p, y, w, self.thresholds)):
            acc += v

    def result(self):
        tp, fp, tn, fn = self.tp, self.fp, self.tn, self.fn
        if self.curve == "PR" and self.summation_method == "interpolation":
            dtp = tp[:-1] - tp[1:]                                         # [KERAS] AUC.interpolate_pr_auc
            p = tp + fp
            dp = p[:-1] - p[1:]
            prec_slope = _div(dtp, np.maximum(dp, 0))
            intercept = tp[1:] - prec_slope * p[1:]
            safe_p_ratio = np.where((p[:-1] > 0) & (p[1:] > 0), _div(p[:-1], np.maximum(p[1:], 0)), 1.0)
            return float(np.sum(_div(prec_slope * (dtp + intercept * np.log(safe_p_ratio)), np.maximum(tp[1:] + fn[1:], 0))))
        recall = _div(tp, tp + fn)
        x, yv = (_div(fp, fp + tn), recall) if self.curve == "ROC" else (recall, _div(tp, tp + fp))
        if self.summation_method == "interpolation":
            h = (yv[:-1] + yv[1:]) / 2.0
        elif self.summation_method == "minoring":
            h = np.minimum(yv[:-1], yv[1:])
        else:
            h = np.maximum(yv[:-1], yv[1:])
        return float(np.sum((x[:-1] - x[1:]) * h))


class _AtThreshold:
    def __init__(self, thresholds=0.5):
        self.t = np.asarray([np.float32(thresholds)], np.float64)
        self.tp = self.fp = self.fn = 0.0

    def update(self, z, y, w=None):
        tp, fp, _, fn = confusion(z, y, w, self.t)
        self.tp += tp[0]; self.fp += fp[0]; self.fn += fn[0]


class Precision(_AtThreshold):
    """[KERAS] keras.metrics.Precision: divide_no_nan(TP, TP + FP) at the threshold (a float32 constant)."""

    def result(self):
        return float(_div(self.tp, self.tp + self.fp))


class Recall(_AtThreshold):
    """[KERAS] keras.metrics.Recall: divide_no_nan(TP, TP + FN) at the threshold (a float32 constant)."""

    def result(self):
        return float(_div(self.tp, self.tp + self.fn))


def for_metric(m):
    """The oracle of a dib_b200.metrics object (or of its resolved kind)."""
    from dib_b200 import metrics as M
    if isinstance(m, M.AUC):
        return AUC(m.num_thresholds, m.curve, m.summation_method, m.from_logits)
    if isinstance(m, M.Precision):
        return Precision(m.threshold)
    if isinstance(m, M.Recall):
        return Recall(m.threshold)
    return Mean(m.kind, threshold=m.threshold, from_logits=m.from_logits)
