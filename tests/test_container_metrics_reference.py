"""CPU checks of the container-metrics restatement (tests/container_metrics_reference.py) and of the finisher that turns the
engine's raw results into scikit-learn's values (sagemaker_xgboost_container_b200/container_metrics.py)."""
import importlib.util
import os
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import container_metrics_reference as R  # noqa: E402
import reference_stubs  # noqa: E402
from sagemaker_xgboost_container_b200 import container_metrics as CM  # noqa: E402

CLASS_NAMES = ["accuracy", "balanced_accuracy", "f1", "f1_binary", "f1_macro", "precision", "precision_macro", "precision_micro",
               "recall", "recall_macro", "recall_micro"]
REG_NAMES = ["mse", "rmse", "mae", "r2"]


class _Labels:
    def __init__(self, y):
        self.y = np.asarray(y, np.float32)

    def get_label(self):
        return self.y


def _run(fn, *args):
    """(value or exception (type, message), [(category, message)] of the warnings)."""
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        try:
            out = fn(*args)
        except Exception as e:          # noqa: BLE001
            out = (type(e), str(e))
    return out, [(w.category, str(w.message)) for w in caught]


def _same(a, b):
    if isinstance(a, float) and isinstance(b, float):
        return (np.isnan(a) and np.isnan(b)) or a == b
    return a == b


@pytest.mark.parametrize("n", list(range(1, 301)) + [8191, 8192, 8193, 8200, 65535, 65536, 65537, 65545, (1 << 20) - 1, 1 << 20, (1 << 20) + 9])
def test_pairwise_sum_matches_numpy(n):
    rng = np.random.default_rng(n)
    a = (rng.standard_normal(n) * rng.choice([1e-3, 1.0, 1e4], n)).astype(np.float32)
    assert R.pairwise_sum(a) == np.sum(a)
    sq = (a * a).astype(np.float32)
    assert R.pairwise_sum(sq) == np.sum(sq)
    assert R.pairwise_sum(sq) == np.sum(sq.reshape(-1, 1), axis=0)[0]       # scikit-learn sums (n, 1) columns


@pytest.mark.parametrize("n", [1, 2, 7, 8, 127, 128, 129, 1000, 8193, 65537, 300001, (1 << 24) + 3])
def test_regression_restatement_matches_sklearn(n):
    rng = np.random.default_rng(7 + n)
    y = (rng.standard_normal(n) * 3 + 1).astype(np.float32)
    p = (y + rng.standard_normal(n).astype(np.float32) * 0.5).astype(np.float32)
    for name in REG_NAMES:
        host, hw = _run(lambda: R.CUSTOM_METRICS[name](p, _Labels(y))[1])
        if name == "r2" and n < 2:
            assert np.isnan(host) and hw
            continue
        assert host == R.regression_restated(name, y, p), name
        d = (y - p).astype(np.float32)
        dev = (y - R.mean32(R.pairwise_sum(y), n)).astype(np.float32)
        fin = CM.finish_regression(name, n, R.pairwise_sum(d * d), R.pairwise_sum(np.abs(d)), R.pairwise_sum(y), R.pairwise_sum(dev * dev), True)
        assert fin == host, name


def test_regression_degenerate():
    y = np.full(50, 2.5, np.float32)
    for p, want in ((y.copy(), 1.0), (y + 1, 0.0)):      # perfect predictions; constant labels
        assert R.CUSTOM_METRICS["r2"](p, _Labels(y))[1] == want
        d = (y - p).astype(np.float32)
        assert CM.finish_regression("r2", 50, np.sum(d * d), np.sum(np.abs(d)), np.sum(y), np.float32(0), True) == want
    assert CM.finish_regression("r2", 1, np.float32(1), np.float32(1), np.float32(1), np.float32(0), True) is CM._UNDECIDED
    assert CM.finish_regression("mse", 10, np.float32(np.inf), np.float32(1), np.float32(1), np.float32(0), True) is CM._UNDECIDED


def _counts(y, pc, P, L=64):
    c = np.zeros((L, P), np.int64)
    np.add.at(c, (y.astype(np.int64), pc), 1)
    return c


def _class_cases():
    rng = np.random.default_rng(3)
    yield "binary", rng.integers(0, 2, 500), rng.integers(0, 2, 500), 2
    yield "multiclass", rng.integers(0, 5, 1000), rng.integers(0, 5, 1000), 5
    yield "never_predicted", rng.integers(0, 5, 300), rng.choice([0, 1, 3], 300), 5
    yield "all_one_pred", rng.integers(0, 2, 100), np.ones(100, np.int64), 2            # every row class 1 (binary:logistic)
    yield "all_zero_pred", rng.integers(0, 2, 100), np.zeros(100, np.int64), 2          # zero division in precision
    yield "one_class", np.ones(40, np.int64), rng.integers(0, 2, 40), 2
    yield "one_class_zero", np.zeros(40, np.int64), np.zeros(40, np.int64), 2
    yield "labels_0_2", rng.choice([0, 2], 200), rng.integers(0, 2, 200), 2            # multi:softmax collapsed to {0, 1}
    yield "labels_0_2_only", rng.choice([0, 2], 200), rng.choice([0, 2], 200), 3
    yield "single_row", np.array([1]), np.array([0]), 2
    yield "k10", rng.integers(0, 10, 2000), rng.integers(0, 10, 2000), 10
    yield "label_63", rng.choice([0, 63], 50), rng.integers(0, 2, 50), 2


@pytest.mark.parametrize("case", list(_class_cases()), ids=lambda c: c[0])
@pytest.mark.parametrize("name", CLASS_NAMES)
def test_class_finisher_matches_sklearn(name, case):
    _, y, pc, P = case
    y = np.asarray(y); pc = np.asarray(pc)
    if P == 2:
        preds = (pc > 0).astype(np.float32)              # 1-D: the class is prediction > 0
    else:
        preds = np.eye(P, dtype=np.float32)[pc]          # 2-D: argmax
    host, hw = _run(lambda: R.CUSTOM_METRICS[name](preds, _Labels(y))[1])
    raw = np.zeros(8 + 64 * 64, np.int64)
    raw[:4] = [1, len(y), P, 64]
    raw[8:8 + 64 * P] = _counts(y, pc, P).ravel()
    dev, dw = _run(lambda: CM.finish(name, raw))
    if isinstance(host, tuple):                          # scikit-learn raised: the finisher must leave it undecided
        assert dev is CM._UNDECIDED
        return
    assert dev is not CM._UNDECIDED, (name, host)
    assert _same(dev, host) and type(dev) is type(host), (dev, host)
    assert dw == hw


def test_class_finisher_empty_and_undecided():
    raw = np.zeros(8 + 64 * 64, np.int64)
    raw[:4] = [0, 0, 2, 64]
    assert CM.finish("accuracy", raw) == 0.0             # no predictions scores 0.0 before any label is read
    assert CM.finish("mse", raw) is CM._UNDECIDED
    raw[:4] = [2, 10, 2, 64]                             # the engine flagged the labels
    assert CM.finish("f1", raw) is CM._UNDECIDED


def _real_container_module():
    path = os.path.join(reference_stubs.REFERENCE_SRC, "sagemaker_xgboost_container", "metrics", "custom_metrics.py")
    if not os.path.exists(path):
        pytest.skip("the container's sources are not present")
    spec = importlib.util.spec_from_file_location(CM.CONTAINER_MODULE, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_restatement_equals_container():
    mod = _real_container_module()
    assert sorted(mod.CUSTOM_METRICS) == sorted(R.CUSTOM_METRICS)
    rng = np.random.default_rng(11)
    y2 = rng.integers(0, 2, 300).astype(np.float32)
    y5 = rng.integers(0, 5, 300).astype(np.float32)
    cases = [(y2, rng.standard_normal(300).astype(np.float32)), (y2, rng.random(300).astype(np.float32)),
             (y5, rng.random((300, 5)).astype(np.float32)), (y5, rng.integers(0, 5, 300).astype(np.float32)),
             (rng.standard_normal(300).astype(np.float32), rng.standard_normal(300).astype(np.float32)),
             (y2, np.zeros(0, np.float32))]
    for y, p in cases:
        for name in CLASS_NAMES + REG_NAMES:
            a = _run(lambda: mod.CUSTOM_METRICS[name](p, _Labels(y)))
            b = _run(lambda: R.CUSTOM_METRICS[name](p, _Labels(y)))
            if isinstance(a[0], tuple) and isinstance(a[0][0], type):
                assert a[0][0] is b[0][0], (name, a, b)
            else:
                assert a[0][0] == b[0][0] and _same(a[0][1], b[0][1]), (name, a, b)
            assert a[1] == b[1], name


def test_recognition_fires_on_the_container_closure(monkeypatch):
    mod = _real_container_module()
    monkeypatch.setitem(sys.modules, CM.CONTAINER_MODULE, mod)
    names = ["accuracy", "rmse", "f1", "r2"]
    fn = mod.configure_feval(names)
    assert CM.recognise(fn) == names
    assert CM.recognise(lambda p, d: fn(p, d)) is None
    assert CM.recognise(R.configure_feval(names)) is None          # same shape, another module
    assert CM.recognise(mod.configure_feval(["accuracy", "nope"])) is None


def test_recognition_on_the_restatement(monkeypatch):
    monkeypatch.setitem(sys.modules, CM.CONTAINER_MODULE, R)
    names = list(R.CUSTOM_METRICS)
    assert CM.recognise(R.configure_feval(names)) == names
    assert CM.recognise(lambda p, d: R.configure_feval(names)(p, d)) is None
    monkeypatch.delitem(sys.modules, CM.CONTAINER_MODULE)
    assert CM.recognise(R.configure_feval(names)) is None
