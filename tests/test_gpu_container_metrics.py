"""The container's own metrics on the GPU (DESIGN.md "Container metrics"): `custom_metric=configure_feval(names)` takes the
device route and reports exactly what the host route (the same closure wrapped in a lambda) reports."""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import container_metrics_reference as R  # noqa: E402
from util import synth  # noqa: E402

pytestmark = pytest.mark.gpu

ALL = list(R.CUSTOM_METRICS)
REG = ["mse", "rmse", "mae", "r2"]
MULTI_SAFE = ["accuracy", "balanced_accuracy", "f1", "f1_macro", "precision_macro", "precision_micro", "recall_macro", "recall_micro"]


@pytest.fixture
def container(monkeypatch, xgb):
    from sagemaker_xgboost_container_b200 import container_metrics as CM
    mod = sys.modules.get(CM.CONTAINER_MODULE)
    if mod is None:
        monkeypatch.setitem(sys.modules, CM.CONTAINER_MODULE, R)
        mod = R
    return mod


def _train(xgb, params, dtrain, evals, rounds, fn, margin=False, **kw):
    res = {}
    out = io.StringIO()
    metric = {"feval": fn} if margin else {"custom_metric": fn}
    with redirect_stdout(out):
        bst = xgb.train(params, dtrain, rounds, evals=evals, evals_result=res, verbose_eval=True, **metric, **kw)
    return bst, res, out.getvalue()


def _custom(res, log, names):
    """The container metrics' part of evals_result (values as repr, so nan equals nan) and of the log lines.  The engine's
    own metric (set so its name differs from every container name) is left out: its double sums may differ in the last
    bits from run to run."""
    hist = {d: {m: [repr(v) for v in vals] for m, vals in ms.items() if m in names} for d, ms in res.items()}
    lines = ["\t".join(f for f in line.split("\t") if f.split(":")[0].partition("-")[2] in names) for line in log.splitlines()]
    return hist, lines


def _bits(v):
    return "nan" if np.isnan(v) else np.float64(v).tobytes()


def raw_checker(xgb, evals, fn, names, margin, log=None):
    """A callback comparing, after every round, the device route's values on the live booster (its prediction cache as the
    round left it) with the container's function on predict(), bit for bit; `log` collects the device values."""
    from sagemaker_xgboost_container_b200 import container_metrics as CM

    class RawEqual(xgb.callback.TrainingCallback):
        def after_iteration(self, model, epoch, evals_log):
            for d, name in evals:
                dev = CM.evaluate(model, d, names, margin)
                host = fn(model.predict(d, training=False, output_margin=margin), d)
                assert [k for k, _ in dev] == [k for k, _ in host]
                for (k, a), (_, b) in zip(dev, host):
                    assert _bits(a) == _bits(b), (epoch, name, k, a, b)
                if log is not None:
                    log.append([_bits(v) for _, v in dev])
            return False
    return RawEqual()


def _check(xgb, mod, params, dtrain, evals, names, rounds=3, margin=False, no_predict=True, **kw):
    from sagemaker_xgboost_container_b200 import container_metrics as CM
    fn = mod.configure_feval(names)
    assert CM.recognise(fn) == names
    orig = xgb.Booster.predict
    if no_predict:
        def refuse(*a, **k):
            raise AssertionError("the device route called Booster.predict")
        xgb.Booster.predict = refuse
    try:
        bst, res_dev, log_dev = _train(xgb, params, dtrain, evals, rounds, fn, margin, **kw)
    finally:
        xgb.Booster.predict = orig
    # the host route, with the raw values of both routes compared on the live booster after every round
    cb = raw_checker(xgb, evals, fn, names, margin)
    _, res_host, log_host = _train(xgb, params, dtrain, evals, rounds, lambda p, d: fn(p, d), margin, callbacks=[cb], **kw)
    assert _custom(res_dev, log_dev, names) == _custom(res_host, log_host, names)
    return bst, res_dev


def _bin(n, seed=0, F=8):
    return synth(n, F, seed, kind="bin")


FAMILIES = [
    ("reg:squarederror", {"eval_metric": "mphe"}, "reg3", REG + MULTI_SAFE),
    ("reg:logistic", {"eval_metric": "logloss"}, "bin", ALL),
    ("binary:logistic", {}, "bin", ALL),
    ("binary:logitraw", {}, "bin", ALL),
    ("binary:hinge", {}, "bin", ALL),
    ("multi:softprob", {"num_class": 3}, "multi3", MULTI_SAFE),
    ("multi:softprob", {"num_class": 10}, "multi10", MULTI_SAFE),
    ("multi:softmax", {"num_class": 3}, "multi3", MULTI_SAFE + REG),
    ("multi:softmax", {"num_class": 10}, "multi10", MULTI_SAFE + REG),
    ("binary:logistic", {"booster": "dart", "rate_drop": 0.3}, "bin", ALL),
    ("binary:logitraw", {"booster": "dart", "rate_drop": 0.5}, "bin", ALL),
    # metrics far above 1: one float32 ulp of a dart margin would show in the log line
    ("reg:squarederror", {"booster": "dart", "rate_drop": 0.5, "eval_metric": "mphe"}, "regbig", REG),
    ("binary:logistic", {"num_parallel_tree": 3, "subsample": 0.8, "colsample_bynode": 0.8}, "bin", ALL),
]


def _data(kind, n, seed):
    if kind == "bin":
        return _bin(n, seed)
    if kind == "regbig":
        X, y = synth(n, 8, seed, kind="reg")
        return X, (y * 300 + 1000).astype(np.float32)
    if kind == "reg3":
        X, y = synth(n, 8, seed, kind="reg")
        return X, np.clip(np.round(y + 1), 0, 2).astype(np.float32)
    K = int(kind[5:])
    return synth(n, 8, seed, kind="multi", K=K)


@pytest.mark.parametrize("n", [1, 7, 8, 127, 128, 129, 8193])
@pytest.mark.parametrize("fam", FAMILIES, ids=lambda f: f[0] + "-" + "-".join("%s%s" % kv for kv in f[1].items()))
def test_device_route_equals_host_route(xgb, container, fam, n):
    obj, extra, kind, names = fam
    X, y = _data(kind, 3000, 1)
    Xv, yv = _data(kind, n, 2)
    dtrain, dval = xgb.DMatrix(X, label=y), xgb.DMatrix(Xv, label=yv)
    params = dict(objective=obj, tree_method="hist", max_depth=4, eta=0.3, **extra)
    # r2 on one row is nan with scikit-learn's warning: left to the container's function, which reads predict()
    _check(xgb, container, params, dtrain, [(dtrain, "train"), (dval, "validation")], names, no_predict=not (n < 2 and "r2" in names))


@pytest.mark.parametrize("n,names", [(1_000_000, ["accuracy", "f1", "precision_macro", "rmse", "mae", "r2"]), (20_000_000, ["accuracy", "rmse", "r2"])])
def test_large_row_counts(xgb, container, n, names):
    X, y = _bin(n, 5, F=4)
    d = xgb.DMatrix(X, label=y)
    params = dict(objective="binary:logistic", tree_method="hist", max_depth=4, eta=0.3)
    _check(xgb, container, params, d, [(d, "train")], names, rounds=2 if n < 10_000_000 else 1)


def test_quantile_dmatrix_base_margin_weights_and_margin_mode(xgb, container):
    X, y = _bin(5000, 3)
    Xv, yv = _bin(3001, 4)
    dtrain = xgb.QuantileDMatrix(X, label=y, weight=np.linspace(0.5, 2, 5000, dtype=np.float32))
    dq = xgb.QuantileDMatrix(Xv, label=yv, ref=dtrain)
    dbm = xgb.DMatrix(Xv, label=yv, base_margin=np.linspace(-1, 1, 3001, dtype=np.float32), weight=np.full(3001, 3.0, np.float32))
    params = dict(objective="binary:logistic", tree_method="hist", max_depth=4, eta=0.3)
    evals = [(dtrain, "train"), (dq, "quantile"), (dbm, "margin")]
    _check(xgb, container, params, dtrain, evals, ALL)
    _check(xgb, container, params, dtrain, evals, ALL, margin=True)
    Xm, ym = _data("multi3", 4000, 6)
    dm = xgb.DMatrix(Xm, label=ym)
    _check(xgb, container, dict(objective="multi:softprob", num_class=3, max_depth=4), dm, [(dm, "train")], MULTI_SAFE, margin=True)


@pytest.mark.parametrize("case", ["continuous_accuracy", "multiclass_f1_binary", "rmse_2d", "label_nan"])
def test_error_paths_match(xgb, container, case):
    if case == "continuous_accuracy":
        X, y = synth(2000, 8, 1, kind="reg"); params, names = dict(objective="reg:squarederror"), ["rmse", "accuracy"]
    elif case == "multiclass_f1_binary":
        X, y = _data("multi3", 2000, 1); params, names = dict(objective="multi:softprob", num_class=3), ["accuracy", "f1_binary"]
    elif case == "rmse_2d":
        X, y = _data("multi3", 2000, 1); params, names = dict(objective="multi:softprob", num_class=3), ["f1", "rmse"]
    else:
        X, y = _bin(2000, 1); params, names = dict(objective="binary:logistic"), ["mae", "accuracy"]
    dtrain = xgb.DMatrix(X, label=y)
    Xv, yv = X[:500], y[:500].copy()
    if case == "label_nan":
        yv[3] = np.nan
    dval = xgb.DMatrix(Xv, label=yv)
    fn = container.configure_feval(names)
    errs = []
    for f in (fn, lambda p, d: fn(p, d)):
        with pytest.raises(Exception) as ei:
            _train(xgb, dict(params, max_depth=3), dtrain, [(dtrain, "train"), (dval, "validation")], 2, f)
        errs.append((type(ei.value), str(ei.value)))
    assert errs[0] == errs[1]


def test_early_stopping_on_f1(xgb, container):
    X, y = _bin(20000, 8)
    Xv, yv = _bin(4000, 9)
    dtrain, dval = xgb.DMatrix(X, label=y), xgb.DMatrix(Xv, label=yv)
    params = dict(objective="binary:logitraw", max_depth=6, eta=0.5)
    fn = container.configure_feval(["accuracy", "f1"])
    kw = dict(early_stopping_rounds=3, maximize=True)
    b1, r1, l1 = _train(xgb, params, dtrain, [(dtrain, "train"), (dval, "validation")], 40, fn, **kw)
    b2, r2, l2 = _train(xgb, params, dtrain, [(dtrain, "train"), (dval, "validation")], 40, lambda p, d: fn(p, d), **kw)
    assert _custom(r1, l1, ["accuracy", "f1"]) == _custom(r2, l2, ["accuracy", "f1"])
    assert b1.best_iteration == b2.best_iteration
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())


def test_deterministic(xgb, container):
    X, y = _bin(300_001, 10)
    d = xgb.DMatrix(X, label=y)
    params = dict(objective="reg:squarederror", max_depth=5, eval_metric="mphe")
    fn = container.configure_feval(ALL)
    runs = []
    for _ in range(2):
        raw = []
        _train(xgb, params, d, [(d, "train")], 3, fn, callbacks=[raw_checker(xgb, [(d, "train")], fn, ALL, False, raw)])
        runs.append(raw)
    assert len(runs[0]) == 3 and runs[0] == runs[1]


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks(xgb, tmp_path):
    """Each rank evaluates its own shard (no all-reduce): its device-route values equal its host-route values bit for bit."""
    import json
    import subprocess
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "cm")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29637", os.path.join(root, "tests", "helpers", "container_metrics_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    vals = []
    for k in range(2):
        with open(out + ".%d.json" % k) as f:
            got = json.load(f)
        assert got["rounds"] == 3 and got["device"] == got["host"]
        vals.append(got["device"])
    assert vals[0] != vals[1]          # two shards, two values: nothing is averaged across ranks
