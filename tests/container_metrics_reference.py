"""Restatement of the container's own metrics (sagemaker_xgboost_container.metrics.custom_metrics) from their behaviour,
plus numpy's float32 pairwise summation and the float32 regression metrics written out in terms of it.

The module has the container's shape: one function per metric name, `CUSTOM_METRICS` mapping names to them and
`configure_feval(names)` returning a closure over `custom_metric_list`.  The GPU tests install it under the container's module
name where the container itself is absent, so the device route recognises it like the real closure.
"""
import numpy as np
from sklearn import metrics as _skm


def class_labels(preds):
    """2-D predictions: np.argmax per row (first maximum, a NaN first); 1-D: 1 where the prediction is above 0."""
    if isinstance(preds[0], np.ndarray):
        return np.argmax(preds, axis=-1)
    return (preds > 0.0).astype(int)


def _classification(score, preds, dtrain):
    if preds.size == 0:
        return 0.0
    return score(dtrain.get_label(), class_labels(preds))


def _make_class_metric(name, score):
    def metric(preds, dtrain):
        return name, _classification(score, preds, dtrain)
    metric.__name__ = name
    return metric


def _make_reg_metric(name, score):
    def metric(preds, dtrain):
        return name, score(dtrain.get_label(), preds)
    metric.__name__ = name
    return metric


accuracy = _make_class_metric("accuracy", _skm.accuracy_score)
balanced_accuracy = _make_class_metric("balanced_accuracy", _skm.balanced_accuracy_score)
f1 = _make_class_metric("f1", lambda y, p: _skm.f1_score(y, p, average="macro"))
f1_binary = _make_class_metric("f1_binary", lambda y, p: _skm.f1_score(y, p, average="binary"))
f1_macro = _make_class_metric("f1_macro", lambda y, p: _skm.f1_score(y, p, average="macro"))
precision = _make_class_metric("precision", _skm.precision_score)
precision_macro = _make_class_metric("precision_macro", lambda y, p: _skm.precision_score(y, p, average="macro"))
precision_micro = _make_class_metric("precision_micro", lambda y, p: _skm.precision_score(y, p, average="micro"))
recall = _make_class_metric("recall", _skm.recall_score)
recall_macro = _make_class_metric("recall_macro", lambda y, p: _skm.recall_score(y, p, average="macro"))
recall_micro = _make_class_metric("recall_micro", lambda y, p: _skm.recall_score(y, p, average="micro"))
mse = _make_reg_metric("mse", _skm.mean_squared_error)
rmse = _make_reg_metric("rmse", _skm.root_mean_squared_error)
mae = _make_reg_metric("mae", _skm.mean_absolute_error)
r2 = _make_reg_metric("r2", _skm.r2_score)

CUSTOM_METRICS = {f.__name__: f for f in (accuracy, balanced_accuracy, f1, f1_binary, f1_macro, mse, rmse, mae, precision,
                                           precision_macro, precision_micro, r2, recall, recall_macro, recall_micro)}


def configure_feval(custom_metric_list):
    def custom_feval(preds, dtrain):
        return [CUSTOM_METRICS[name](preds, dtrain) for name in custom_metric_list]
    return custom_feval


# ---------------------------------------------------------------------------------------------------------------------
# numpy's float32 pairwise sum and the float32 regression metrics in its terms
# ---------------------------------------------------------------------------------------------------------------------
def pairwise_sum(a):
    """np.sum of a 1-D float32 array: blocks of at most 128 terms with eight strided accumulators (fewer than 8 terms: in
    sequence from 0), larger ranges split at n/2 - (n/2 mod 8) and the halves added."""
    a = np.asarray(a, np.float32)
    n = len(a)
    if n < 8:
        res = np.float32(0)
        for x in a:
            res = np.float32(res + x)
        return res
    if n <= 128:
        m = n - n % 8
        r = a[:m].reshape(-1, 8)
        acc = r[0].copy()
        for row in r[1:]:
            acc = (acc + row).astype(np.float32)
        res = np.float32(np.float32(np.float32(acc[0] + acc[1]) + np.float32(acc[2] + acc[3]))
                         + np.float32(np.float32(acc[4] + acc[5]) + np.float32(acc[6] + acc[7])))
        for x in a[m:]:
            res = np.float32(res + x)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return np.float32(pairwise_sum(a[:n2]) + pairwise_sum(a[n2:]))


def mean32(total, n):
    """numpy's float32 mean: the float32 sum divided by the count in double, rounded to float32."""
    return np.float32(np.float64(total) / np.float64(n))


def regression_restated(name, y, p):
    y, p = np.asarray(y, np.float32), np.asarray(p, np.float32)
    n = len(y)
    d = (y - p).astype(np.float32)
    if name in ("mse", "rmse"):
        v = mean32(pairwise_sum(d * d), n)
        return float(np.sqrt(v)) if name == "rmse" else float(v)
    if name == "mae":
        return float(mean32(pairwise_sum(np.abs(d)), n))
    num = pairwise_sum(d * d)
    dev = (y - mean32(pairwise_sum(y), n)).astype(np.float32)
    den = pairwise_sum(dev * dev)
    if num == 0:
        return 1.0
    if den == 0:
        return 0.0
    return float(np.float32(1) - num / den)
