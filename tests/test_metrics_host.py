"""CPU: the float64 Keras metric oracle (tests/metrics_oracle.py) against scikit-learn and closed forms, the host half of the
compiled metrics (dib_b200.metrics: parsing, names, order, refusals, and the values of a metric tail) against the oracle."""
import numpy as np
import pytest
from sklearn import metrics as skm

from dib_b200 import metrics as M
from tests import metrics_oracle as MO


def _data(n, seed, weights=True):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal(n) * 2
    y = (rng.uniform(size=n) < sigmoid_np(z + rng.standard_normal(n))).astype(np.float64)
    w = rng.uniform(0, 50, n) if weights else None
    if weights:
        w[rng.choice(n, n // 10, replace=False)] = 0.0
    return z, y, w


def sigmoid_np(z):
    return 1.0 / (1.0 + np.exp(-z))


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs scikit-learn
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("weights", [False, True])
def test_mean_metrics_match_sklearn(weights):
    rng = np.random.default_rng(1)
    n = 500
    z, y = rng.standard_normal((n, 6)), rng.standard_normal((n, 6))
    w = rng.uniform(0, 50, n) if weights else None
    for kind, ref in (("mse", skm.mean_squared_error), ("mae", skm.mean_absolute_error)):
        m = MO.Mean(kind)
        m.update(z[:200], y[:200], None if w is None else w[:200])           # epoch-stateful: two batches, one value
        m.update(z[200:], y[200:], None if w is None else w[200:])
        assert abs(m.result() - ref(y, z, sample_weight=w)) < 1e-12 * max(1.0, abs(m.result()))
    # crossentropy on logits is exactly the log loss of sigmoid(z) / softmax(z)
    zb, yb, wb = _data(n, 2, weights)
    bce = MO.Mean("binary_crossentropy", from_logits=True)
    bce.update(zb, yb, wb)
    assert abs(bce.result() - skm.log_loss(yb, sigmoid_np(zb), sample_weight=wb)) < 1e-12
    z3 = rng.standard_normal((n, 3)) * 2
    y3 = rng.integers(0, 3, n).astype(np.float64)
    sce = MO.Mean("sparse_categorical_crossentropy", from_logits=True)
    sce.update(z3, y3, w)
    soft = np.exp(z3 - z3.max(1, keepdims=True))
    soft /= soft.sum(1, keepdims=True)
    assert abs(sce.result() - skm.log_loss(y3, soft, sample_weight=w, labels=[0, 1, 2])) < 1e-12
    # on probabilities Keras adds eps inside the log: |log(p + eps) - log p| <= eps / p, so within eps / min p of the log loss
    p = np.clip(sigmoid_np(zb), 0.01, 0.99)
    bp = MO.Mean("binary_crossentropy")
    bp.update(p, yb, wb)
    assert abs(bp.result() - skm.log_loss(yb, p, sample_weight=wb)) < MO.EPSILON / 0.01
    sp = MO.Mean("sparse_categorical_crossentropy")
    sp.update(soft, y3, w)
    assert abs(sp.result() - skm.log_loss(y3, soft, sample_weight=w, labels=[0, 1, 2])) < 1e-6
    acc = MO.Mean("binary_accuracy", threshold=0.3)
    acc.update(p, yb, wb)
    assert abs(acc.result() - skm.accuracy_score(yb, p > 0.3, sample_weight=wb)) < 1e-12
    sacc = MO.Mean("sparse_categorical_accuracy")
    sacc.update(z3, y3, w)
    assert abs(sacc.result() - skm.accuracy_score(y3, z3.argmax(1), sample_weight=w)) < 1e-12


@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("t", [0.5, 0.25, 0.9])
def test_precision_recall_match_sklearn(t, weights):
    z, y, w = _data(3000, 3, weights)
    p = sigmoid_np(z)
    pr, rc = MO.Precision(t), MO.Recall(t)
    for o in (pr, rc):
        o.update(p[:1000], y[:1000], None if w is None else w[:1000])
        o.update(p[1000:], y[1000:], None if w is None else w[1000:])
    pred = p > np.float32(t)
    assert abs(pr.result() - skm.precision_score(y, pred, sample_weight=w)) < 1e-12
    assert abs(rc.result() - skm.recall_score(y, pred, sample_weight=w)) < 1e-12


def _bucket_weights(p, y, w, thresholds):
    """Weights of the positive and negative rows per bucket b = number of thresholds p exceeds."""
    b = (p[:, None] > thresholds[None, :]).sum(1)
    w = np.ones(len(p)) if w is None else w
    T = len(thresholds)
    pos = np.bincount(b[y != 0], w[y != 0], minlength=T + 1)
    neg = np.bincount(b[y == 0], w[y == 0], minlength=T + 1)
    return neg, pos


@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("T", [200, 17, 2])
def test_roc_auc_matches_sklearn_within_the_discretisation_bound(T, weights):
    """With T thresholds a (positive, negative) pair is ordered correctly unless both rows fall in the same bucket (then it
    counts 1/2 in the trapezoids, 0, 1/2 or 1 in the exact AUC): |AUC_T - AUC| <= sum_b pos_b neg_b / (2 P N)."""
    z, y, w = _data(4000, 4, weights)
    p = sigmoid_np(z)
    a = MO.AUC(T)
    a.update(z[:1500], y[:1500], None if w is None else w[:1500])
    a.update(z[1500:], y[1500:], None if w is None else w[1500:])
    exact = skm.roc_auc_score(y, p, sample_weight=w)
    a_logits = MO.AUC(T, from_logits=True)
    a_logits.update(z, y, w)
    a_probs = MO.AUC(T)
    a_probs.update(p, y, w)
    assert a_logits.result() == a_probs.result()
    neg, pos = _bucket_weights(p, y, w, MO.auc_thresholds(T))
    bound = (pos * neg).sum() / (2 * pos.sum() * neg.sum())
    err = abs(a_probs.result() - exact)
    print(f"[metrics] ROC AUC, T = {T}: |AUC_T - AUC| = {err:.3e} <= {bound:.3e}")
    assert err <= bound + 1e-12


@pytest.mark.parametrize("weights", [False, True])
def test_roc_auc_is_exact_when_scores_sit_on_thresholds(weights):
    T = 51
    t = MO.auc_thresholds(T)
    rng = np.random.default_rng(5)
    n = 2000
    p = t[rng.integers(1, T - 1, n)]
    y = (rng.uniform(size=n) < p).astype(np.float64)
    w = rng.uniform(0, 5, n) if weights else None
    a = MO.AUC(T)
    a.update(p, y, w)
    assert abs(a.result() - skm.roc_auc_score(y, p, sample_weight=w)) < 1e-12


@pytest.mark.parametrize("curve", ["ROC", "PR"])
def test_auc_closed_forms(curve):
    n = 400
    y = np.r_[np.zeros(n // 2), np.ones(n // 2)]
    sep = np.r_[np.linspace(0.05, 0.4, n // 2), np.linspace(0.6, 0.95, n // 2)]
    # (PR minoring: precision is 0 / 0 -> 0 above the highest score, and min() takes that zero for the last recall step)
    for method in ("interpolation", "minoring", "majoring") if curve == "ROC" else ("interpolation", "majoring"):
        a = MO.AUC(200, curve, method)
        a.update(sep, y)
        assert abs(a.result() - 1.0) < 1e-12, (curve, method)
    if curve == "ROC":
        for method in ("interpolation", "minoring", "majoring"):
            r = MO.AUC(200, curve, method)
            r.update(sep[::-1], y)
            assert abs(r.result()) < 1e-12
        e = MO.AUC(200)
        e.update(np.full(n, 0.3), y)
        assert abs(e.result() - 0.5) < 1e-12
    else:
        # PR of all-equal scores: the precision of the whole set, P / n, from recall 0 to 1
        e = MO.AUC(200, "PR", "interpolation")
        e.update(np.full(n, 0.3), y)
        assert abs(e.result() - 0.5) < 1e-12


@pytest.mark.parametrize("kind", ["mse", "mae", "binary_accuracy", "binary_crossentropy", "auc", "auc_pr", "precision", "recall"])
def test_integer_weights_equal_repeated_rows(kind):
    z, y, _ = _data(300, 6, False)
    p = sigmoid_np(z)
    w = np.random.default_rng(6).integers(0, 5, 300).astype(np.float64)
    make = {"auc": lambda: MO.AUC(), "auc_pr": lambda: MO.AUC(curve="PR"), "precision": lambda: MO.Precision(),
            "recall": lambda: MO.Recall()}.get(kind, lambda: MO.Mean(kind))
    a, b = make(), make()
    a.update(p, y, w)
    rep = np.repeat(np.arange(300), w.astype(int))
    b.update(p[rep], y[rep])
    assert abs(a.result() - b.result()) < 1e-12 * max(1.0, abs(b.result()))


# ---------------------------------------------------------------------------------------------------------------------
# dib_b200.metrics: the values of a metric tail, parsing, names, order, refusals
# ---------------------------------------------------------------------------------------------------------------------
def _tail_from_rows(entries, z, y, w):
    """The metric tail the kernel writes, restated on the host in float64 (bucket b = thresholds p exceeds, p and the
    thresholds in float32)."""
    tail = np.zeros(M.tail_length(entries))
    for e in entries:
        if not e.in_tail:
            continue
        we = w if (e.weighted and w is not None) else np.ones(len(z))
        m = e.metric
        if m.kind != "confusion":
            v = MO.ROW_FUNCTIONS[m.kind](z, y, dict(threshold=m.threshold, from_logits=m.from_logits))
            tail[e.offset:e.offset + 2] = [np.sum(we * v), np.sum(we)]
            continue
        T = m.num_thresholds
        thr = MO.auc_thresholds(T) if T > 1 else np.asarray([np.float32(m.threshold)], np.float64)
        zz = np.asarray(z, np.float64).reshape(-1)
        p = (MO.sigmoid(zz) if m.from_logits else zz).astype(np.float32).astype(np.float64)
        neg, pos = _bucket_weights(p, np.asarray(y).reshape(-1), we, thr)
        tail[e.offset:e.offset + e.size] = np.r_[neg, pos]
    return tail


def test_metric_values_of_a_tail_equal_the_oracle():
    z, y, w = _data(5000, 7)
    y = y[:, None]
    p = sigmoid_np(z)[:, None].astype(np.float32).astype(np.float64)           # the model's fp32 outputs
    objs = [M.AUC(name="roc"), M.AUC(curve="PR", name="pr"), M.AUC(57, summation_method="minoring", name="a57"),
            M.AUC(33, summation_method="majoring", name="a33"),
            M.Precision(0.3), M.Recall(0.7), M.BinaryAccuracy(threshold=0.4), M.MeanSquaredError(), M.MeanAbsoluteError(),
            M.BinaryCrossentropy()]
    entries = M.compile_metrics(objs, [M.AUC(from_logits=False), "mse"], "bce_probs", 1, "sigmoid")
    vals = M.metric_values(entries, _tail_from_rows(entries, p, y, w))
    for e in entries:
        ref = MO.for_metric(e.metric)
        ref.update(p, y, w if e.weighted else None)
        assert abs(vals[e.name] - ref.result()) < 1e-12 * max(1.0, abs(ref.result())), e.name
    # the epoch value sums the tails of its batches
    half = _tail_from_rows(entries, p[:2000], y[:2000], w[:2000]) + _tail_from_rows(entries, p[2000:], y[2000:], w[2000:])
    vals2 = M.metric_values(entries, half)
    for k in vals:
        assert abs(vals2[k] - vals[k]) < 1e-12 * max(1.0, abs(vals[k]))


def test_sparse_metrics_values_of_a_tail_equal_the_oracle():
    rng = np.random.default_rng(8)
    z = rng.standard_normal((700, 3)).astype(np.float32).astype(np.float64)
    y = rng.integers(0, 3, 700).astype(np.float64)
    w = rng.uniform(0, 3, 700)
    entries = M.compile_metrics(["sparse_categorical_crossentropy", M.SparseCategoricalCrossentropy(from_logits=True, name="sce"),
                                 "accuracy", "sparse_categorical_accuracy"], ["accuracy"], "sparse_ce_logits", 3, None)
    vals = M.metric_values(entries, _tail_from_rows(entries, z, y, w))
    assert [e.name for e in entries] == ["sparse_categorical_crossentropy", "sce", "accuracy", "sparse_categorical_accuracy",
                                         "weighted_accuracy"]
    ref = MO.Mean("sparse_categorical_crossentropy", from_logits=True)
    ref.update(z, y)
    assert abs(vals["sce"] - ref.result()) < 1e-12
    ref = MO.Mean("sparse_categorical_accuracy")
    ref.update(z, y, w)
    assert abs(vals["weighted_accuracy"] - ref.result()) < 1e-12


def test_names_order_and_weighted_prefix():
    e = M.compile_metrics(["mae", "accuracy", M.AUC(from_logits=True, name="roc"), "acc"],
                          ["mae", M.Precision(name="p"), "accuracy", "binary_crossentropy"], "bce_logits", 1, "sigmoid")
    assert [x.name for x in e] == ["mae", "accuracy", "roc", "accuracy", "weighted_mae", "p", "weighted_accuracy",
                                   "binary_crossentropy"]
    assert [x.weighted for x in e] == [False] * 4 + [True] * 4
    assert [x.in_tail for x in e] == [True, False, True, False, True, True, True, True]
    assert e[-1].metric.from_logits is False                      # the string is Keras' function as written
    assert isinstance(e[6].metric, M.BinaryAccuracy) and e[6].metric.threshold == 0.5
    offs = [(x.offset, x.size) for x in e if x.in_tail]
    assert offs == [(0, 2), (2, 402), (404, 2), (406, 4), (410, 2), (412, 2)]
    assert M.tail_length(e) == 414
    assert [x.name for x in M.compile_metrics(["mse", "mean_squared_error"], None, "mse", 6, None)] == ["mse",
                                                                                                        "mean_squared_error"]
    assert M.compile_metrics(None, None, "mse", 6, None) == [] and M.compile_metrics(["accuracy"], [], "external", 1, None)
    assert M.signature(M.compile_metrics(["accuracy"], None, "bce_logits", 1, None)) == ()


@pytest.mark.parametrize("metrics,weighted,loss,out,act,match", [
    ([lambda yt, yp: yp], None, "bce_logits", 1, None, "callables"),
    (["f1"], None, "bce_logits", 1, None, "unknown metric"),
    (["mse"], None, "infonce", 8, None, "infonce"),
    (None, ["mae"], "external", 1, None, "external"),
    ([M.AUC()], None, "bce_logits", 1, None, "AUC\\(from_logits=True\\)"),
    ([M.Precision()], None, "bce_logits", 1, None, "output_activation_fn='sigmoid'"),
    ([M.Recall()], None, "mse", 1, "relu", "logits"),
    ([M.AUC(from_logits=True)], None, "mse", 3, None, "multi-class AUC"),
    ([M.Precision()], None, "bce_probs", 2, "sigmoid", "one output"),
    (["sparse_categorical_accuracy"], None, "bce_logits", 1, None, "class-label"),
    (["mse"], None, "sparse_ce_logits", 3, None, "class labels"),
    ([M.AUC(from_logits=True), M.AUC(from_logits=True)], None, "bce_logits", 1, None, "distinct names"),
    (["mse"], [M.MeanSquaredError(name="mse")], "mse", 1, None, None),
    ([M.MeanSquaredError(name="loss")], None, "mse", 1, None, "distinct names"),
    ([M.AUC(1500, from_logits=True), M.AUC(600, from_logits=True, name="a2")], None, "bce_logits", 1, None, "thresholds"),
    (["mse"] * 9, ["mae"] * 8, "mse", 1, None, None),
    ("mse", None, "mse", 1, None, "list"),
])
def test_refusals(metrics, weighted, loss, out, act, match):
    if match is None:            # accepted: a duplicate across the lists is prefixed; 17 entries with distinct names
        if len(metrics) > 1:
            objs = [M.MeanSquaredError(name=f"m{i}") for i in range(9)] + [M.MeanAbsoluteError(name=f"a{i}") for i in range(8)]
            with pytest.raises(ValueError, match="at most 16"):
                M.compile_metrics(objs, None, loss, out, act)
        else:
            assert [e.name for e in M.compile_metrics(metrics, weighted, loss, out, act)] == ["mse", "weighted_mse"]
        return
    with pytest.raises(ValueError, match=match):
        M.compile_metrics(metrics, weighted, loss, out, act)


def test_metric_objects_refuse_what_is_not_implemented():
    for make in (lambda: M.AUC(multi_label=True), lambda: M.AUC(num_labels=3), lambda: M.AUC(thresholds=[0.5]),
                 lambda: M.AUC(num_thresholds=1), lambda: M.AUC(curve="XY"), lambda: M.AUC(summation_method="x"),
                 lambda: M.Precision(thresholds=[0.2, 0.4]), lambda: M.Precision(top_k=1), lambda: M.Recall(class_id=0),
                 lambda: M.Recall(thresholds=1.5), lambda: M.BinaryCrossentropy(label_smoothing=0.1),
                 lambda: M.MeanSquaredError(dtype="float16")):
        with pytest.raises(ValueError):
            make()
    assert M.AUC().name == "auc" and M.Precision().name == "precision" and M.Recall().name == "recall"
    assert M.MeanSquaredError().name == "mean_squared_error" and M.AUC(name="x").name == "x"
    import dib_b200
    assert dib_b200.keras_compat.metrics.AUC is M.AUC and dib_b200.metrics.metrics.Recall is M.Recall
