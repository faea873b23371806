"""aucpr and one-vs-rest multi-class auc / aucpr on the GPU, against tests/auc_reference.py applied to predict() at every
round: binary and multi-class objectives, weights, row counts from 1 to millions, determinism, the degenerate and
invalid inputs, scratch reuse, the container's early-stopping and log paths, and a two-rank run."""
import math
import os
import re

import numpy as np
import pytest

import auc_reference as AR

pytestmark = pytest.mark.gpu

BINARY = ["binary:logistic", "binary:logitraw", "reg:squarederror"]
MULTI = ["multi:softprob", "multi:softmax"]
SIZES = [1, 1000, 70_000, 2_000_000]
# 3M rows are 1465 tiles of 2048, more than the 8 CTAs per SM of the curve kernels' grid on a 132-SM H100: some CTAs walk
# several tiles
BINARY_SIZES = SIZES + [3_000_000]


def _data(n, seed, K=0, weighted=False):
    """Few distinct feature values, so shallow trees give heavily tied scores."""
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 8, (n, 3)).astype(np.float32)
    if K:
        logits = X[:, :1] * np.arange(K, dtype=np.float32) * 0.3 - X[:, 1:2] * 0.2
        y = np.argmax(logits + rng.gumbel(size=(n, K)) * 2.0, axis=1).astype(np.float32)
    else:
        y = (X[:, 0] + X[:, 1] * 0.5 + rng.standard_normal(n) * 2.0 > 5.0).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    return X, y, w


def _close(got, want):
    if math.isnan(want):
        return math.isnan(got)
    return got == pytest.approx(want, rel=1e-12, abs=1e-15)


def _train(xgb, params, d, rounds, **kw):
    res = {}
    bst = xgb.train(params, d, rounds, evals=[(d, "validation")], evals_result=res, verbose_eval=False, **kw)
    return bst, res["validation"]


def _binary_want(p, y, w):
    try:
        return AR.aucpr(p, y, w)
    except ValueError:
        return None


@pytest.mark.parametrize("n", BINARY_SIZES)
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("objective", BINARY)
def test_binary_aucpr_every_round(xgb, objective, weighted, n):
    X, y, w = _data(n, 1 + n % 97, weighted=weighted)
    d = xgb.DMatrix(X, label=y, weight=w)
    params = {"objective": objective, "max_depth": 2, "eta": 0.5, "eval_metric": ["aucpr"]}
    if _binary_want(np.zeros(n, np.float32), y, w) is None:          # one class only: raises like binary auc
        with pytest.raises(xgb.XGBoostError, match="only contains pos or neg"):
            _train(xgb, params, d, 1)
        return
    rounds = 4
    bst, log = _train(xgb, params, d, rounds)
    assert len(log["aucpr"]) == rounds
    for r in range(rounds):
        p = bst.predict(d, iteration_range=(0, r + 1))
        want = AR.aucpr(p, y, w)
        assert _close(log["aucpr"][r], want), (objective, n, r, log["aucpr"][r], want)


@pytest.mark.parametrize("weighted", [False, True])
def test_binary_aucpr_imbalanced_every_round(xgb, weighted):
    """About one positive in a thousand and more than ten thousand tie blocks (a base margin of ~12.7k levels, so the scores do
    not collapse onto the few leaves the rare positives let the trees grow): late PR segments have b / a near N / P, where a
    plain difference of two logs would lose the 1e-12 agreement."""
    rng = np.random.default_rng(31 + weighted)
    n = 1_000_000
    X = rng.integers(0, 64, (n, 4)).astype(np.float32)
    z = X[:, 0] / 64.0 + X[:, 1] / 128.0 - X[:, 2] / 256.0 + rng.standard_normal(n) * 0.35
    y = (z > np.quantile(z, 0.999)).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    d = xgb.DMatrix(X, label=y, weight=w, base_margin=(np.round(z * 4000) / 4000 - 7.0).astype(np.float32))
    rounds = 5
    bst, log = _train(xgb, {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "eval_metric": ["aucpr"]}, d, rounds)
    blocks = []
    for r in range(rounds):
        p = bst.predict(d, iteration_range=(0, r + 1))
        blocks.append(len(np.unique(p)))
        want = AR.aucpr(p, y, w)
        assert _close(log["aucpr"][r], want), (weighted, r, log["aucpr"][r], want)
    assert max(blocks) > 10_000, blocks


def test_unlabelled_aft_matrix_raises(xgb):
    """survival:aft reads bounds; a matrix that has no label gets an error from auc / aucpr, not a read of missing labels."""
    rng = np.random.default_rng(41)
    X = rng.standard_normal((2000, 3)).astype(np.float32)
    lo = rng.uniform(1.0, 5.0, 2000).astype(np.float32)
    d = xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=lo * 1.5)
    for m in ("aucpr", "auc"):
        with pytest.raises(xgb.XGBoostError, match="labels are not correctly provided"):
            xgb.train({"objective": "survival:aft", "eval_metric": m}, d, 1, evals=[(d, "v")], verbose_eval=False)
    # the booster stays usable: the same matrix evaluates its own metric afterwards
    bst = xgb.train({"objective": "survival:aft", "eval_metric": "aft-nloglik"}, d, 2, evals=[(d, "v")], verbose_eval=False)
    assert bst.num_boosted_rounds() == 2


def _probs(xgb, params, d, rounds, bst):
    """predict()'s probabilities at every round: multi:softmax predicts labels, so its softprob twin (the same trees, bit for
    bit) gives them."""
    if params["objective"] == "multi:softprob":
        return bst
    twin = xgb.train(dict(params, objective="multi:softprob"), d, rounds, verbose_eval=False)
    np.testing.assert_array_equal(twin.predict(d, output_margin=True).view(np.uint32), bst.predict(d, output_margin=True).view(np.uint32))
    return twin


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("K", [3, 10])
@pytest.mark.parametrize("objective", MULTI)
def test_multiclass_auc_aucpr_every_round(xgb, objective, K, weighted, n):
    if n >= 2_000_000 and objective == "multi:softmax" and K == 3:
        pytest.skip("covered by multi:softprob at this size")
    X, y, w = _data(n, 7 + K + n % 89, K=K, weighted=weighted)
    d = xgb.DMatrix(X, label=y, weight=w)
    params = {"objective": objective, "num_class": K, "max_depth": 2, "eta": 0.5, "eval_metric": ["auc", "aucpr"]}
    rounds = 3
    bst, log = _train(xgb, params, d, rounds)
    src = _probs(xgb, params, d, rounds, bst)
    for r in range(rounds):
        p = src.predict(d, iteration_range=(0, r + 1)).reshape(n, K)
        pieces = AR.class_pieces(p, y, w)
        want_auc, want_pr = AR.multiclass_auc(p, y, w, pieces), AR.multiclass_aucpr(p, y, w, pieces)
        assert _close(log["auc"][r], want_auc), (objective, K, n, r, log["auc"][r], want_auc)
        assert _close(log["aucpr"][r], want_pr), (objective, K, n, r, log["aucpr"][r], want_pr)
    if n == 1:
        assert math.isnan(log["auc"][0]) and math.isnan(log["aucpr"][0])


def test_deterministic(xgb):
    lines = []
    for _ in range(2):
        X, y, w = _data(300_000, 5, K=4, weighted=True)
        d = xgb.DMatrix(X, label=y, weight=w)
        bst = xgb.train({"objective": "multi:softprob", "num_class": 4, "max_depth": 3, "eval_metric": ["auc", "aucpr"]}, d, 3, verbose_eval=False)
        Xb, yb, wb = _data(300_000, 6, weighted=True)
        db = xgb.DMatrix(Xb, label=yb, weight=wb)
        bb = xgb.train({"objective": "binary:logistic", "max_depth": 3, "eval_metric": ["aucpr"]}, db, 3, verbose_eval=False)
        lines.append(bst.eval_set([(d, "v")], 3) + bb.eval_set([(db, "v")], 3))
    assert lines[0] == lines[1]


def test_absent_class_is_nan_and_early_stopping_runs(xgb):
    X, y, _ = _data(5000, 11, K=3)
    y[y == 2] = 0                       # class 2 never appears
    d = xgb.DMatrix(X, label=y)
    params = {"objective": "multi:softprob", "num_class": 3, "max_depth": 2, "eval_metric": ["auc", "aucpr"]}
    bst, log = _train(xgb, params, d, 20, early_stopping_rounds=3)
    assert all(math.isnan(v) for v in log["auc"]) and all(math.isnan(v) for v in log["aucpr"])
    assert bst.num_boosted_rounds() <= 20


def test_invalid_inputs(xgb):
    X, y, _ = _data(1000, 12)
    one = xgb.DMatrix(X, label=np.ones(1000, np.float32))
    with pytest.raises(xgb.XGBoostError, match="only contains pos or neg"):
        xgb.train({"objective": "binary:logistic", "eval_metric": "aucpr"}, one, 1, evals=[(one, "v")], verbose_eval=False)
    y2 = y.copy()
    y2[3] = 2.0
    bad = xgb.DMatrix(X, label=y2)
    with pytest.raises(xgb.XGBoostError, match=r"label must be in \[0, 1\] for aucpr"):
        xgb.train({"objective": "reg:squarederror", "eval_metric": "aucpr"}, bad, 1, evals=[(bad, "v")], verbose_eval=False)
    grouped = xgb.DMatrix(X, label=y, group=[500, 500])
    with pytest.raises(xgb.XGBoostError, match="ranking PR-AUC"):
        xgb.train({"objective": "rank:pairwise", "eval_metric": "aucpr"}, grouped, 1, evals=[(grouped, "v")], verbose_eval=False)
    q = xgb.DMatrix(X, label=y)
    for m in ("auc", "aucpr"):
        with pytest.raises(xgb.XGBoostError, match="reg:quantileerror model with 2 outputs"):
            xgb.train({"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "eval_metric": m}, q, 1, evals=[(q, "v")], verbose_eval=False)


def test_no_device_memory_growth(xgb):
    import torch
    X, y, _ = _data(1_000_000, 13, K=5)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train({"objective": "multi:softprob", "num_class": 5, "max_depth": 2, "eval_metric": ["auc", "aucpr"]}, d, 2, verbose_eval=False)
    Xb, yb, _ = _data(1_000_000, 14)
    db = xgb.DMatrix(Xb, label=yb)
    bb = xgb.train({"objective": "binary:logistic", "max_depth": 2, "eval_metric": ["aucpr"]}, db, 2, verbose_eval=False)
    first = bst.eval_set([(d, "v")], 2) + bb.eval_set([(db, "v")], 2)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(50):
        assert bst.eval_set([(d, "v")], 2) + bb.eval_set([(db, "v")], 2) == first
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def test_container_paths(xgb):
    X, y, w = _data(20_000, 15, weighted=True)
    Xv, yv, _ = _data(5000, 16)
    d, dv = xgb.DMatrix(X, label=y, weight=w), xgb.DMatrix(Xv, label=yv)
    res = {}
    bst = xgb.train({"objective": "binary:logistic", "max_depth": 3, "eta": 0.3, "eval_metric": ["aucpr"]}, d, 60,
                    evals=[(d, "train"), (dv, "validation")], evals_result=res, early_stopping_rounds=5, verbose_eval=False)
    hist = res["validation"]["aucpr"]
    assert bst.best_iteration == int(np.argmax(hist))
    # the container's tuning regex for validation:aucpr (the #011 of the CloudWatch line is this tab)
    line = bst.eval_set([(dv, "validation")], 0)
    m = re.match(r".*\[[0-9]+\].*\tvalidation-aucpr:(\S+)", line)
    assert m and float(m.group(1)) == pytest.approx(AR.aucpr(bst.predict(dv), yv), rel=1e-12)
    clf = xgb.XGBClassifier(n_estimators=5, max_depth=2, eval_metric="aucpr")
    clf.fit(Xv, yv.astype(int), eval_set=[(Xv, yv.astype(int))], verbose=False)
    assert len(clf.evals_result()["validation_0"]["aucpr"]) == 5


def two_rank_data():
    X, y, w = _data(40_000, 21, K=3, weighted=True)
    Xb, yb, wb = _data(40_000, 22, weighted=True)
    return X, y, w, Xb, yb, wb


TWO_RANK_MULTI = {"objective": "multi:softprob", "num_class": 3, "max_depth": 2, "eval_metric": ["auc", "aucpr"]}
TWO_RANK_BINARY = {"objective": "binary:logistic", "max_depth": 2, "eval_metric": ["aucpr"]}


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks(xgb, tmp_path):
    """Each rank evaluates its half: multi-class auc follows the all-reduced per-class sums, aucpr the mean of the ranks."""
    import subprocess
    import sys
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "auc")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29631", os.path.join(root, "tests", "helpers", "auc_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y, w, Xb, yb, wb = two_rank_data()
    half = len(y) // 2
    parts = [slice(0, half), slice(half, None)]
    shards, pr_vals, bin_vals = [], [], []
    for k, sl in enumerate(parts):
        p = np.load(out + ".%d.npz" % k)
        shards.append((p["multi"], y[sl], w[sl]))
        pr_vals.append(AR.multiclass_aucpr(p["multi"], y[sl], w[sl]))
        bin_vals.append(AR.binary_aucpr(p["binary"], yb[sl], wb[sl]))
    with open(out + ".eval") as f:
        got = dict(kv.split(":") for kv in f.read().split("\t")[1:])
    assert _close(float(got["m-auc"]), AR.ranks_multiclass_auc(shards))
    assert _close(float(got["m-aucpr"]), AR.ranks_aucpr(pr_vals))
    assert _close(float(got["b-aucpr"]), AR.ranks_aucpr(bin_vals))
