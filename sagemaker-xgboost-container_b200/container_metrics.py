"""The container's own metrics on the GPU (DESIGN.md "Container metrics").

`sagemaker_xgboost_container.metrics.custom_metrics` evaluates accuracy, f1, precision, recall, ... and scikit-learn's mse /
rmse / mae / r2 outside xgboost: `train()` receives `custom_metric=configure_feval(names)`, which for every eval set in every
round would predict the whole model again, copy the predictions and labels to the host and run scikit-learn there.  When the
metric callable is that very closure, `Booster.eval_set` asks the engine for exact raw results from the prediction cache
instead (integer confusion counts; float32 sums in numpy's pairwise order) and finishes them here with scikit-learn's own
rules.  Whatever the engine leaves undecided, and whatever the finisher cannot certify, runs the container's function on
`predict()` as before, so values, warnings and exceptions are the container's.
"""
import math
import sys
import warnings

import numpy as np

from .backend import get_backend

CONTAINER_MODULE = "sagemaker_xgboost_container.metrics.custom_metrics"

_CLASS_METRICS = {
    # name -> (scikit-learn function name, average)
    "accuracy": ("accuracy_score", None), "balanced_accuracy": ("balanced_accuracy_score", None),
    "f1": ("f1_score", "macro"), "f1_binary": ("f1_score", "binary"), "f1_macro": ("f1_score", "macro"),
    "precision": ("precision_score", None), "precision_macro": ("precision_score", "macro"),
    "precision_micro": ("precision_score", "micro"),
    "recall": ("recall_score", None), "recall_macro": ("recall_score", "macro"), "recall_micro": ("recall_score", "micro"),
}
_REG_METRICS = ("mse", "rmse", "mae", "r2")
_DECIDED_CLASS, _DECIDED_REG, _DECIDED_LABEL_SUMS = 1, 2, 4
_HEAD = 8
_UNDECIDED = object()


def recognise(fn):
    """The metric names when `fn` is the container's `configure_feval(names)` closure over metrics this module finishes,
    else None (any other callable keeps the host route)."""
    mod = sys.modules.get(CONTAINER_MODULE)
    if mod is None or getattr(fn, "__globals__", None) is not getattr(mod, "__dict__", None):
        return None
    try:
        if fn.__code__ is not mod.configure_feval([]).__code__:
            return None
        cells = dict(zip(fn.__code__.co_freevars, fn.__closure__ or ()))
        names = list(cells["custom_metric_list"].cell_contents)
        table = mod.CUSTOM_METRICS
        for name in names:
            if not isinstance(name, str) or (name not in _CLASS_METRICS and name not in _REG_METRICS):
                return None
            if table[name] is not getattr(mod, name):
                return None
    except Exception:
        return None
    return names


def evaluate(booster, dmat, names, output_margin):
    """[(name, value)] for the names in order, as the container's closure returns them."""
    mod = sys.modules[CONTAINER_MODULE]
    raw = get_backend().booster_eval_container_metrics(booster.handle, dmat.handle, names, output_margin)
    preds = None
    out = []
    for name in names:
        value = finish(name, raw)
        if value is _UNDECIDED:
            if preds is None:
                preds = booster.predict(dmat, training=False, output_margin=output_margin)
            out.append(mod.CUSTOM_METRICS[name](preds, dmat))
        else:
            out.append((name, value))
    return out


def device_route_available():
    return hasattr(get_backend(), "booster_eval_container_metrics")


def finish(name, raw):
    """scikit-learn's value of metric `name` from the engine's raw result, or _UNDECIDED."""
    decided, n, P, L = (int(v) for v in raw[:4])
    if name in _CLASS_METRICS:
        if n == 0:
            return 0.0                   # compute_multiclass_and_binary_metrics: no predictions scores 0.0
        if not decided & _DECIDED_CLASS:
            return _UNDECIDED
        return _finish_class(name, raw[_HEAD:_HEAD + L * P].reshape(L, P))
    if not decided & _DECIDED_REG or n == 0:
        return _UNDECIDED
    sums = raw[4:8].astype(np.uint32).view(np.float32)
    return finish_regression(name, n, sums[0], sums[1], sums[2], sums[3], bool(decided & _DECIDED_LABEL_SUMS))


def _finish_class(name, counts):
    """scikit-learn on the distinct (label, predicted class) pairs weighted by their counts: the same value and the same
    warnings as on the rows themselves (tests/test_container_metrics_reference.py); an exception leaves it undecided."""
    import sklearn.metrics as skm
    labels, preds = np.nonzero(counts)
    fn_name, average = _CLASS_METRICS[name]
    kwargs = {} if average is None else {"average": average}
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        try:
            value = getattr(skm, fn_name)(labels.astype(np.float32), preds.astype(np.int64),
                                          sample_weight=counts[labels, preds].astype(np.float64), **kwargs)
        except Exception:
            return _UNDECIDED
    for w in caught:
        warnings.warn_explicit(w.message, w.category, w.filename, w.lineno, registry=_registry)
    return value


_registry = {}


def _mean(total, n):
    # numpy's float32 mean: the float32 sum divided by the count in double, rounded to float32
    return np.float32(np.float64(total) / np.float64(n))


def finish_regression(name, n, sum_sq, sum_abs, sum_y, sum_dev, label_sums):
    """scikit-learn's float32 mean_squared_error / root_mean_squared_error / mean_absolute_error / r2_score from the pairwise
    sums, or _UNDECIDED where scikit-learn would warn (an overflow, r2 on fewer than two rows)."""
    sum_sq, sum_abs = np.float32(sum_sq), np.float32(sum_abs)
    if name in ("mse", "rmse"):
        if not math.isfinite(sum_sq):
            return _UNDECIDED
        mse = _mean(sum_sq, n)
        return float(np.sqrt(mse)) if name == "rmse" else float(mse)
    if name == "mae":
        return float(_mean(sum_abs, n)) if math.isfinite(sum_abs) else _UNDECIDED
    if not label_sums or n < 2 or not (math.isfinite(sum_sq) and math.isfinite(sum_y) and math.isfinite(sum_dev)):
        return _UNDECIDED
    num, den = sum_sq, np.float32(sum_dev)
    if num == 0:
        return 1.0
    if den == 0:
        return 0.0
    return float(np.float32(1) - num / den)
