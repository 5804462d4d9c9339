"""Compiled Keras metrics: ``model.compile(metrics=[...], weighted_metrics=[...])`` beyond ``'accuracy'``.

The metric objects below describe Keras 2 metrics; the CUDA library sums each one over the rows of a step into the metric
tail of the statistics vector (``dib_set_metrics`` in include/dib_b200.h), the tail rides the data-parallel all-reduce, an
epoch's tails are summed on the device in float64, and :func:`metric_values` turns the sums into the values Keras reports.

    mean metrics       value = sum_i w_i m_i / sum_i w_i over every row of the epoch (Keras' stateful Mean; 0 when sum w = 0)
    AUC                Keras' evenly spaced thresholds {-1e-7, 1/(T-1), ..., 1 + 1e-7}, a row is positive at t when p > t,
                       ROC / PR curves with the interpolation, minoring or majoring sums of keras.metrics.AUC.result
    Precision, Recall  TP / (TP + FP) and TP / (TP + FN) at their threshold (0 when the denominator is 0)

``w_i`` is the step's sample weight (``sample_weight`` times the ``class_weight`` map in training) for a metric listed in
``weighted_metrics`` and 1 for one listed in ``metrics``.  ``'accuracy'`` (or ``'acc'``) in ``metrics`` keeps the
statistics slot it always had and is reported as ``accuracy``.
"""
from __future__ import annotations

import numpy as np

from . import _lib

MAX_METRICS = 16               # DIB_MAX_METRICS
MAX_BUCKETS = 2048             # DIB_MAX_METRIC_BUCKETS: sum over the AUC / Precision / Recall metrics of (thresholds + 1)


class Metric:
    """A compiled metric: ``kind`` (a key of ``_lib.METRIC_KINDS``), its parameters and its history ``name``."""
    kind = None
    from_logits = False
    threshold = 0.0
    num_thresholds = 0

    def __init__(self, name=None, dtype=None):
        if dtype not in (None, "float32"):
            raise ValueError(f"{type(self).__name__}: only dtype float32 is implemented, got {dtype!r}")
        self.name = name if name is not None else self.default_name

    def __repr__(self):
        return f"<{type(self).__name__} {self.name!r}>"

    def get_config(self):
        """The constructor arguments that rebuild this metric (``type(m)(**m.get_config())``)."""
        return {"name": self.name}


class BinaryAccuracy(Metric):
    """keras.metrics.BinaryAccuracy: mean over the outputs of [(z > threshold) == y]."""
    kind, default_name = "binary_accuracy", "binary_accuracy"

    def __init__(self, name=None, dtype=None, threshold=0.5):
        super().__init__(name, dtype)
        self.threshold = float(threshold)

    def get_config(self):
        return dict(super().get_config(), threshold=self.threshold)


class SparseCategoricalAccuracy(Metric):
    """keras.metrics.SparseCategoricalAccuracy: [argmax z == y] (the string ``'sparse_categorical_accuracy'``)."""
    kind, default_name = "sparse_categorical_accuracy", "sparse_categorical_accuracy"


class MeanSquaredError(Metric):
    """keras.metrics.MeanSquaredError: mean over the outputs of (z - y)^2."""
    kind, default_name = "mse", "mean_squared_error"


class MeanAbsoluteError(Metric):
    """keras.metrics.MeanAbsoluteError: mean over the outputs of |z - y|."""
    kind, default_name = "mae", "mean_absolute_error"


class BinaryCrossentropy(Metric):
    """keras.metrics.BinaryCrossentropy: keras.backend.binary_crossentropy averaged over the outputs; from_logits=False clips
    p to [1e-7, 1 - 1e-7]."""
    kind, default_name = "binary_crossentropy", "binary_crossentropy"

    def __init__(self, name=None, dtype=None, from_logits=False, label_smoothing=0):
        super().__init__(name, dtype)
        if label_smoothing:
            raise ValueError("BinaryCrossentropy(label_smoothing=...) is not implemented")
        self.from_logits = bool(from_logits)

    def get_config(self):
        return dict(super().get_config(), from_logits=self.from_logits)


class SparseCategoricalCrossentropy(Metric):
    """keras.metrics.SparseCategoricalCrossentropy: keras.backend.sparse_categorical_crossentropy; from_logits=False clips p
    to [1e-7, 1 - 1e-7] and normalises it."""
    kind, default_name = "sparse_categorical_crossentropy", "sparse_categorical_crossentropy"

    def __init__(self, name=None, dtype=None, from_logits=False, axis=-1):
        super().__init__(name, dtype)
        if axis != -1:
            raise ValueError("SparseCategoricalCrossentropy(axis=...) other than -1 is not implemented")
        self.from_logits = bool(from_logits)

    def get_config(self):
        return dict(super().get_config(), from_logits=self.from_logits)


class _Confusion(Metric):
    kind = "confusion"


class AUC(_Confusion):
    """keras.metrics.AUC for one output: ``num_thresholds`` evenly spaced thresholds, ``curve`` 'ROC' or 'PR',
    ``summation_method`` 'interpolation', 'minoring' or 'majoring'; ``from_logits=True`` applies sigmoid to z first."""
    default_name = "auc"

    def __init__(self, num_thresholds=200, curve="ROC", summation_method="interpolation", name=None, dtype=None,
                 thresholds=None, multi_label=False, num_labels=None, label_weights=None, from_logits=False):
        super().__init__(name, dtype)
        if thresholds is not None:
            raise ValueError("AUC(thresholds=[...]) is not implemented: use num_thresholds (evenly spaced, as Keras' default)")
        if multi_label or num_labels not in (None, 1) or label_weights is not None:
            raise ValueError("multi-label AUC (multi_label, num_labels, label_weights) is not implemented")
        if int(num_thresholds) <= 1:
            raise ValueError("`num_thresholds` must be > 1.")
        if str(curve).upper() not in ("ROC", "PR"):
            raise ValueError(f"Invalid AUC curve value: {curve!r}")
        if str(summation_method).lower() not in ("interpolation", "minoring", "majoring"):
            raise ValueError(f"Invalid AUC summation method value: {summation_method!r}")
        self.num_thresholds = int(num_thresholds)
        self.curve = str(curve).upper()
        self.summation_method = str(summation_method).lower()
        self.from_logits = bool(from_logits)

    def get_config(self):
        return dict(super().get_config(), num_thresholds=self.num_thresholds, curve=self.curve,
                    summation_method=self.summation_method, from_logits=self.from_logits)


class _AtThreshold(_Confusion):
    def __init__(self, thresholds=None, top_k=None, class_id=None, name=None, dtype=None):
        super().__init__(name, dtype)
        if top_k is not None or class_id is not None:
            raise ValueError(f"{type(self).__name__}(top_k=..., class_id=...) is not implemented")
        t = 0.5 if thresholds is None else thresholds
        if isinstance(t, (list, tuple, np.ndarray)):
            raise ValueError(f"{type(self).__name__} takes one threshold here, got {thresholds!r}")
        t = float(t)
        if not 0.0 <= t <= 1.0:
            raise ValueError(f"Threshold values must be in [0, 1]. Received: {t}")
        self.threshold = t
        self.num_thresholds = 1

    def get_config(self):
        return dict(super().get_config(), thresholds=self.threshold)


class Precision(_AtThreshold):
    """keras.metrics.Precision(thresholds=0.5): TP / (TP + FP), a row predicted positive when p > threshold."""
    default_name = "precision"


class Recall(_AtThreshold):
    """keras.metrics.Recall(thresholds=0.5): TP / (TP + FN), a row predicted positive when p > threshold."""
    default_name = "recall"


class metrics:
    """The ``keras.metrics`` namespace of the metrics the engine computes."""
    BinaryAccuracy = BinaryAccuracy
    SparseCategoricalAccuracy = SparseCategoricalAccuracy
    MeanSquaredError = MeanSquaredError
    MeanAbsoluteError = MeanAbsoluteError
    BinaryCrossentropy = BinaryCrossentropy
    SparseCategoricalCrossentropy = SparseCategoricalCrossentropy
    AUC = AUC
    Precision = Precision
    Recall = Recall


def serialize(m):
    """A compiled metric as JSON-able data: ``'accuracy'`` stays the string, an object becomes {class, config}."""
    return m if isinstance(m, str) else {"class": type(m).__name__, "config": m.get_config()}


def deserialize(spec):
    """The inverse of :func:`serialize`."""
    if isinstance(spec, str):
        return spec
    cls = getattr(metrics, spec["class"], None) if isinstance(spec, dict) else None
    if not (isinstance(cls, type) and issubclass(cls, Metric)):
        raise ValueError(f"unknown metric {spec!r}")
    return cls(**spec["config"])


ACCURACY = "accuracy"          # the statistics slot of metrics=['accuracy'] (a compiled entry, not a tail metric)

_STRINGS = {
    "binary_accuracy": lambda: BinaryAccuracy(),
    "sparse_categorical_accuracy": lambda: SparseCategoricalAccuracy(),
    "mse": lambda: MeanSquaredError(name="mse"),
    "mean_squared_error": lambda: MeanSquaredError(name="mean_squared_error"),
    "mae": lambda: MeanAbsoluteError(name="mae"),
    "mean_absolute_error": lambda: MeanAbsoluteError(name="mean_absolute_error"),
    "binary_crossentropy": lambda: BinaryCrossentropy(),
    "sparse_categorical_crossentropy": lambda: SparseCategoricalCrossentropy(),
}


class CompiledMetric:
    """One entry of the compiled metrics, in history order: the accuracy slot, or a tail metric with its weighting and its
    place [offset, offset + size) in the metric tail."""

    def __init__(self, metric, name, weighted):
        self.metric, self.name, self.weighted = metric, name, bool(weighted)
        self.offset = self.size = 0

    @property
    def in_tail(self):
        return self.metric is not ACCURACY

    def spec(self):
        """(kind, weighted, from_logits, num_thresholds, threshold): what the library computes for this entry."""
        m = self.metric
        return (m.kind, int(self.weighted), int(m.from_logits), int(m.num_thresholds), float(m.threshold))


def _resolve(m, loss_kind, weighted):
    """A metric object for one entry of ``metrics`` / ``weighted_metrics``, or ACCURACY for the statistics slot."""
    if isinstance(m, Metric):
        return m
    if isinstance(m, str):
        key = m
        if key in ("accuracy", "acc"):
            if not weighted:
                return ACCURACY
            # the weighted twin of the slot: Keras resolves 'accuracy' from the loss as the slot does
            return (SparseCategoricalAccuracy(name=ACCURACY) if loss_kind == "sparse_ce_logits"
                    else BinaryAccuracy(name=ACCURACY))
        if key in _STRINGS:
            return _STRINGS[key]()
        raise ValueError(f"unknown metric {m!r}: the engine computes 'accuracy', {', '.join(repr(k) for k in _STRINGS)} "
                         "and the objects of dib_b200.metrics")
    if callable(m):
        raise ValueError(f"metric {m!r}: Python callables are not supported as metrics; the engine computes its metrics on the "
                         "device (strings, or the objects of dib_b200.metrics)")
    raise ValueError(f"unsupported metric {m!r}")


def _check(metric, loss_kind, output_dimensionality, output_activation_fn):
    sparse_metric = metric.kind in ("sparse_categorical_accuracy", "sparse_categorical_crossentropy")
    if sparse_metric != (loss_kind == "sparse_ce_logits"):
        raise ValueError(f"metric {metric.name!r}: " + (
            "the sparse categorical metrics need the class-label targets of SparseCategoricalCrossentropy"
            if sparse_metric else
            "with SparseCategoricalCrossentropy the targets are class labels; use 'accuracy', 'sparse_categorical_accuracy' "
            "or 'sparse_categorical_crossentropy'"))
    if metric.kind != "confusion":
        return
    if int(output_dimensionality) != 1:
        raise ValueError(f"metric {metric.name!r}: AUC, Precision and Recall need one output (output_dimensionality=1); "
                         "multi-label and multi-class AUC are not implemented")
    if not metric.from_logits and output_activation_fn != "sigmoid":
        raise ValueError(f"metric {metric.name!r} needs probabilities in [0, 1] (Keras asserts it), but the model outputs "
                         "logits: use AUC(from_logits=True), or output_activation_fn='sigmoid' with a probability loss")


def compile_metrics(metrics, weighted_metrics, loss_kind, output_dimensionality, output_activation_fn):
    """Parse ``compile(metrics=, weighted_metrics=)`` for a model with compiled loss ``loss_kind``: the entries in history
    order (``metrics`` then ``weighted_metrics``, each in the order given), tail offsets assigned.  A weighted metric whose
    name is also an unweighted one's gets the ``weighted_`` prefix.  Raises ValueError on everything the engine does not
    compute."""
    entries = []
    for lst, weighted in ((metrics, False), (weighted_metrics, True)):
        if lst is None:
            continue
        if isinstance(lst, (str, Metric)) or not hasattr(lst, "__iter__"):
            raise ValueError(f"{'weighted_metrics' if weighted else 'metrics'} must be a list, got {lst!r}")
        for m in lst:
            r = _resolve(m, loss_kind, weighted)
            entries.append(CompiledMetric(r, ACCURACY if r is ACCURACY else r.name, weighted))
    tail = [e for e in entries if e.in_tail]
    if tail and loss_kind in ("infonce", "external"):
        raise ValueError(f"the {loss_kind!r} loss computes no metrics on the device: compile it without metrics "
                         "(or with metrics=['accuracy'] for the external loss)")
    for e in tail:
        _check(e.metric, loss_kind, output_dimensionality, output_activation_fn)
    plain = {e.name for e in entries if not e.weighted}
    for e in entries:
        if e.weighted and e.name in plain:
            e.name = "weighted_" + e.name
    names = [e.name for e in entries if e.in_tail or e.weighted]
    seen = set(e.name for e in entries if not e.in_tail and not e.weighted)
    for nm in names:
        if nm in seen or nm in ("loss", "beta") or (nm.startswith("KL") and nm[2:].isdigit()):
            raise ValueError(f"two compiled metrics, or a metric and a statistic, would both be reported as {nm!r}: "
                             "give the metric objects distinct names")
        seen.add(nm)
    if len(tail) > MAX_METRICS:
        raise ValueError(f"at most {MAX_METRICS} metrics besides metrics=['accuracy'] are implemented")
    if sum(e.metric.num_thresholds + 1 for e in tail if e.metric.kind == "confusion") > MAX_BUCKETS:
        raise ValueError(f"AUC / Precision / Recall: at most {MAX_BUCKETS} thresholds plus one per metric in total")
    off = 0
    for e in tail:
        e.offset = off
        e.size = 2 * (e.metric.num_thresholds + 1) if e.metric.kind == "confusion" else 2
        off += e.size
    return entries


def tail_length(entries):
    return sum(e.size for e in entries if e.in_tail)


def library_specs(entries):
    """The ``dib_metric_spec`` array of the tail metrics (and their count) for dib_set_metrics."""
    tail = [e for e in entries if e.in_tail]
    arr = (_lib.DibMetricSpec * max(len(tail), 1))()
    for i, e in enumerate(tail):
        kind, weighted, from_logits, T, threshold = e.spec()
        arr[i] = _lib.DibMetricSpec(_lib.METRIC_KINDS[kind], weighted, from_logits, T, threshold)
    return arr, len(tail)


def confusion_counts(neg, pos):
    """TP, FP, TN, FN at each of the T thresholds from the bucket sums [T + 1] of the negative and positive rows (bucket b:
    p exceeds exactly b thresholds): TP(t_j) = sum_{b > j} pos[b], and so on."""
    neg, pos = np.asarray(neg, np.float64), np.asarray(pos, np.float64)
    tp = np.cumsum(pos[::-1])[::-1][1:]
    fp = np.cumsum(neg[::-1])[::-1][1:]
    return tp, fp, neg.sum() - fp, pos.sum() - tp


def _div_no_nan(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    out = np.zeros(np.broadcast(a, b).shape)
    np.divide(a, b, out=out, where=b != 0)
    return out


def auc_from_counts(tp, fp, tn, fn, curve="ROC", summation_method="interpolation"):
    """keras.metrics.AUC.result on confusion counts over ascending thresholds (float64)."""
    tp, fp, tn, fn = (np.asarray(a, np.float64) for a in (tp, fp, tn, fn))
    if curve == "PR" and summation_method == "interpolation":
        # AUC.interpolate_pr_auc (Davis & Goadrich 2006)
        dtp = tp[:-1] - tp[1:]
        p = tp + fp
        dp = p[:-1] - p[1:]
        prec_slope = _div_no_nan(dtp, np.maximum(dp, 0))
        intercept = tp[1:] - prec_slope * p[1:]
        both = (p[:-1] > 0) & (p[1:] > 0)
        safe_p_ratio = np.where(both, _div_no_nan(p[:-1], np.maximum(p[1:], 0)), 1.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            inc = _div_no_nan(prec_slope * (dtp + intercept * np.log(safe_p_ratio)), np.maximum(tp[1:] + fn[1:], 0))
        return float(inc.sum())
    recall = _div_no_nan(tp, tp + fn)
    if curve == "ROC":
        x, y = _div_no_nan(fp, fp + tn), recall
    else:
        x, y = recall, _div_no_nan(tp, tp + fp)
    if summation_method == "interpolation":
        heights = (y[:-1] + y[1:]) / 2.0
    elif summation_method == "minoring":
        heights = np.minimum(y[:-1], y[1:])
    else:
        heights = np.maximum(y[:-1], y[1:])
    return float(np.sum((x[:-1] - x[1:]) * heights))


def metric_values(entries, tail):
    """{name: value} of the tail metrics from the (summed) tail; the accuracy slot is not in the tail."""
    t = np.asarray(tail, dtype=np.float64)
    out = {}
    for e in entries:
        if not e.in_tail:
            continue
        s = t[e.offset:e.offset + e.size]
        m = e.metric
        if m.kind != "confusion":
            out[e.name] = float(s[0] / s[1]) if s[1] != 0 else 0.0
            continue
        T = m.num_thresholds
        tp, fp, tn, fn = confusion_counts(s[:T + 1], s[T + 1:])
        if isinstance(m, AUC):
            out[e.name] = auc_from_counts(tp, fp, tn, fn, m.curve, m.summation_method)
        elif isinstance(m, Precision):
            out[e.name] = float(_div_no_nan(tp[0], tp[0] + fp[0]))
        else:
            out[e.name] = float(_div_no_nan(tp[0], tp[0] + fn[0]))
    return out


def signature(entries):
    """What a handle and a captured graph depend on: the tail metrics' specs in order (empty without metrics)."""
    return tuple(e.spec() for e in entries if e.in_tail)


__all__ = ["Metric", "BinaryAccuracy", "SparseCategoricalAccuracy", "MeanSquaredError", "MeanAbsoluteError",
           "BinaryCrossentropy", "SparseCategoricalCrossentropy", "AUC", "Precision", "Recall", "metrics",
           "compile_metrics", "metric_values"]
