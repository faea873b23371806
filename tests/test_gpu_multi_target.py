"""Multi-target regression on the GPU (run with `pytest -m gpu` on an H100): gradients against tests/multi_target_reference.py,
the independence of the targets (target j's trees are those of a one-column model on Y[:, j]), T = 1, the intercept and the
metrics, prediction shapes, model IO, other features, QuantileDMatrix batches, the error cases, the sklearn wrapper and two
ranks."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import multi_target_reference as MR
from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
BASE = dict(tree_method="hist", max_bin=256, max_depth=5, eta=0.3)


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _same_bits(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return a.shape == b.shape and bool(np.all((_u32(a) == _u32(b)) | (np.isnan(a) & np.isnan(b))))


def labels3(n, F, seed, objective, missing_frac=0.0):
    """X and a 3-column label suited to the objective: [0, 1] labels for the logistic family, > -1 for squaredlogerror."""
    X, y = synth(n, F, seed, "reg", missing_frac=missing_frac)
    rng = np.random.default_rng(seed + 1)
    Y = np.stack([y, -0.5 * y + 0.3 * rng.standard_normal(n), np.abs(y) + rng.laplace(0, 0.3, n)], axis=1).astype(f32)
    if objective in MR.LOGISTIC:
        Y = (Y > np.median(Y, axis=0)).astype(f32)
        Y[::7, 1] = 0.25                                         # a soft label
    elif objective == "reg:squaredlogerror":
        Y = np.abs(Y).astype(f32)
    return X, np.ascontiguousarray(Y)


def _tree(m, t):
    s, e = int(m["tree_offset"][t]), int(m["tree_offset"][t + 1])
    return {k: m[k][s:e] for k in ("left", "right", "parent", "split_index", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")}


def _same_tree(a, b):
    return all(_same_bits(a[k], b[k]) if a[k].dtype == f32 else np.array_equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------------------- 1 gradients
@pytest.mark.parametrize("objective", MR.OBJECTIVES)
@pytest.mark.parametrize("weighted", [False, True])
def test_gradients(xgb, objective, weighted):
    X, Y = labels3(20011, 6, 1, objective)
    n = len(Y)
    rng = np.random.default_rng(2)
    w = rng.uniform(0, 3, n).astype(f32) if weighted else None
    m = rng.standard_normal((n, 3)).astype(f32)
    m[:40] = Y[:40]                                              # d == 0
    d = xgb.DMatrix(X, label=Y, weight=w)
    for extra in ({}, dict(scale_pos_weight=2.5), dict(subsample=0.5, seed=3)):
        params = dict(BASE, objective=objective, huber_slope=1.5, **extra)
        bst = xgb.Booster(params, [d])                           # kept alive across the call: its handle is freed with it
        got = _be().booster_compute_gradient(bst.handle, d.handle, m, round=2)
        keep = None
        if "subsample" in extra:
            from forest_reference import row_mask
            keep = row_mask(3, 2, 0, n, 0.5)
        ref = MR.gradient(objective, m, Y, w, extra.get("scale_pos_weight", 1.0), 1.5, keep)
        if objective in MR.EXACT:
            assert _same_bits(got, ref), (objective, extra)
        else:                      # a few ulp between CUDA and numpy (module doc); the kernel itself is pinned below
            np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-7)
        # each target's pairs are the single-target kernel's on its label column, bit for bit
        for j in range(3):
            dj = xgb.DMatrix(X, label=Y[:, j], weight=w)
            bj = xgb.Booster(params, [dj])
            one = _be().booster_compute_gradient(bj.handle, dj.handle, m[:, j:j + 1], round=2)
            assert _same_bits(got[:, j], one[:, 0]), (objective, extra, j)


# ---------------------------------------------------------------------------------------------------------------- 2 independence
IND_CASES = {
    "plain": ({}, {}),
    "weights": ({}, dict(weighted=True)),
    "missing": ({}, dict(missing_frac=0.1)),
    "subsample": (dict(subsample=0.7, seed=4), {}),
    "lossguide": (dict(grow_policy="lossguide", max_depth=0, max_leaves=24), {}),
}


@pytest.mark.parametrize("objective", MR.OBJECTIVES)
@pytest.mark.parametrize("case", list(IND_CASES))
def test_targets_are_independent(xgb, objective, case):
    extra, opts = IND_CASES[case]
    X, Y = labels3(12000, 8, 41, objective, opts.get("missing_frac", 0.0))
    w = np.random.default_rng(42).uniform(0.2, 2, len(Y)).astype(f32) if opts.get("weighted") else None
    p = dict(BASE, objective=objective, base_score=0.4, **extra)
    b3 = xgb.train(p, xgb.DMatrix(X, label=Y, weight=w), num_boost_round=3, verbose_eval=False)
    m3 = _be().booster_export_model(b3.handle)
    assert list(m3["tree_info"]) == [0, 1, 2] * 3
    p3 = b3.predict(xgb.DMatrix(X))
    for j in range(3):
        b1 = xgb.train(p, xgb.DMatrix(X, label=Y[:, j], weight=w), num_boost_round=3, verbose_eval=False)
        m1 = _be().booster_export_model(b1.handle)
        for r in range(3):
            assert _same_tree(_tree(m3, 3 * r + j), _tree(m1, r)), (objective, case, j, r)
        assert _same_bits(p3[:, j], b1.predict(xgb.DMatrix(X)))


# ---------------------------------------------------------------------------------------------------------------- 3 T = 1
@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic", "reg:absoluteerror"])
def test_one_column_is_the_1d_label(xgb, objective):
    X, Y = labels3(8000, 6, 51, objective)
    a = xgb.train(dict(BASE, objective=objective), xgb.DMatrix(X, label=Y[:, 0]), num_boost_round=3, verbose_eval=False)
    b = xgb.train(dict(BASE, objective=objective), xgb.DMatrix(X, label=Y[:, :1]), num_boost_round=3, verbose_eval=False)
    assert bytes(a.save_raw("json")) == bytes(b.save_raw("json")) and a.save_config() == b.save_config()
    assert _same_bits(a.predict(xgb.DMatrix(X)), b.predict(xgb.DMatrix(X)))
    assert json.loads(bytes(a.save_raw("json")))["learner"]["learner_model_param"]["num_target"] == "1"


# ---------------------------------------------------------------------------------------------------------------- 4 intercept, metrics
@pytest.mark.parametrize("objective", MR.OBJECTIVES)
def test_intercept(xgb, objective):
    X, Y = labels3(30001, 4, 61, objective)
    for w in (None, np.random.default_rng(62).uniform(0, 4, len(Y)).astype(f32)):
        bst = xgb.train(dict(BASE, objective=objective, scale_pos_weight=1.5), xgb.DMatrix(X, label=Y, weight=w), num_boost_round=1, verbose_eval=False)
        got = f32(_be().booster_export_model(bst.handle)["base_score"])
        ref = MR.intercept(objective, Y, w, scale_pos_weight=1.5)
        # double sums in another order, and expf under the logistic transform: agree to a few float32 ulp
        assert abs(float(got) - float(ref)) <= 4 * float(np.spacing(np.abs(ref))) + 1e-7, (objective, got, ref)
        if objective == "reg:absoluteerror":
            assert got == ref


@pytest.mark.parametrize("objective,metrics", [("reg:squarederror", ["rmse", "mae", "mape", "mphe"]),
                                               ("reg:squaredlogerror", ["rmsle"]),
                                               ("binary:logistic", ["logloss", "error", "error@0.3"]),
                                               ("binary:logitraw", ["logloss", "error"])])
@pytest.mark.parametrize("weighted", [False, True])
def test_metrics(xgb, objective, metrics, weighted):
    X, Y = labels3(20000, 6, 71, objective)
    if objective == "reg:squarederror":
        Y = Y + 3.0                                              # mape divides by the label
    w = np.random.default_rng(72).uniform(0, 2, len(Y)).astype(f32) if weighted else None
    d = xgb.DMatrix(X, label=Y, weight=w)
    res = {}
    bst = xgb.train(dict(BASE, objective=objective, eval_metric=metrics), d, num_boost_round=3, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    pred = bst.predict(d)
    if objective == "binary:logitraw":
        pred = 1.0 / (1.0 + np.exp(-pred.astype(np.float64)))
    for name in metrics:
        assert res["train"][name][-1] == pytest.approx(MR.metric(name, Y, pred, w), rel=2e-5, abs=2e-6), name
    # the default metric is the objective's usual one
    res = {}
    xgb.train(dict(BASE, objective=objective), d, num_boost_round=1, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    assert list(res["train"]) == [{"reg:squarederror": "rmse", "reg:squaredlogerror": "rmsle", "binary:logistic": "logloss", "binary:logitraw": "logloss"}[objective]]


def test_unsupported_metrics_raise(xgb):
    X, Y = labels3(2000, 4, 73, "reg:squarederror")
    d = xgb.DMatrix(X, label=Y)
    for name in ("poisson-nloglik", "quantile", "ndcg", "mse", "merror"):
        with pytest.raises(xgb.core.XGBoostError, match="multi-target"):
            xgb.train(dict(BASE, objective="reg:squarederror", eval_metric=name, quantile_alpha="0.5"), d, num_boost_round=1, evals=[(d, "t")], verbose_eval=False)
    for name in ("auc", "aucpr"):
        with pytest.raises(xgb.core.XGBoostError, match="outputs per row"):
            xgb.train(dict(BASE, objective="reg:squarederror", eval_metric=name), d, num_boost_round=1, evals=[(d, "t")], verbose_eval=False)


# ---------------------------------------------------------------------------------------------------------------- 5 prediction
def test_prediction_shapes_and_ranges(xgb):
    from oracle.gbt_oracle import shap_bruteforce
    X, Y = labels3(3000, 5, 81, "binary:logistic")
    d = xgb.DMatrix(X, label=Y)
    bst = xgb.train(dict(BASE, objective="binary:logistic", max_depth=3), d, num_boost_round=4, verbose_eval=False)
    shp = MR.shapes(3000, 3, 5, 12)
    p, mg = bst.predict(d), bst.predict(d, output_margin=True)
    assert p.shape == shp["value"] and mg.shape == shp["margin"] and bst.predict(d, strict_shape=True).shape == shp["strict_shape"]
    np.testing.assert_allclose(p, 1.0 / (1.0 + np.exp(-mg.astype(np.float64))), rtol=2e-6)        # the sigmoid, element-wise
    assert _same_bits(bst.predict(d, training=True), p)
    leaf = bst.predict(d, pred_leaf=True)
    assert leaf.shape == shp["pred_leaf"]
    np.testing.assert_array_equal(bst[1:3].predict(d, pred_leaf=True), leaf[:, 3:9])
    assert _same_bits(bst[1:3].predict(d, output_margin=True), bst.predict(d, output_margin=True, iteration_range=(1, 3)))
    short = xgb.train(dict(BASE, objective="binary:logistic", max_depth=3), d, num_boost_round=2, verbose_eval=False)
    assert _same_bits(short.predict(d), bst.predict(d, iteration_range=(0, 2)))
    contrib = bst.predict(d, pred_contribs=True)
    assert contrib.shape == shp["pred_contribs"]
    np.testing.assert_allclose(contrib.sum(axis=2), mg, rtol=0, atol=2e-5)
    model = _be().booster_export_model(bst.handle)
    ref = shap_bruteforce(model, X[:200])          # the feature columns; the bias column is checked by the sum above
    np.testing.assert_allclose(contrib[:200, :, :-1], ref[:, :, :-1], rtol=0, atol=2e-5)
    # a (n, T) base_margin
    bm = np.random.default_rng(82).normal(0, 1, (3000, 3)).astype(f32)
    dm = xgb.DMatrix(X, label=Y, base_margin=bm)
    trees = mg - np.float32(np.log(model["base_score"] / (1 - model["base_score"])))
    np.testing.assert_allclose(bst.predict(dm, output_margin=True), trees + bm, rtol=0, atol=2e-5)


# ---------------------------------------------------------------------------------------------------------------- 6 model IO
def test_model_io_round_trips(xgb, tmp_path):
    X, Y = labels3(5000, 6, 91, "reg:pseudohubererror")
    d = xgb.DMatrix(X, label=Y)
    params = dict(BASE, objective="reg:pseudohubererror", max_depth=4)
    bst = xgb.train(params, d, num_boost_round=4, verbose_eval=False)
    p0 = bst.predict(d)
    for fmt in ("json", "ubj"):
        path = str(tmp_path / ("m." + fmt))
        bst.save_model(path)
        assert _same_bits(xgb.Booster(model_file=path).predict(d), p0)
    assert _same_bits(pickle.loads(pickle.dumps(bst)).predict(d), p0)
    doc = json.loads(open(str(tmp_path / "m.json")).read())
    lmp = doc["learner"]["learner_model_param"]
    assert lmp["num_target"] == "3" and lmp["num_class"] == "0"
    assert doc["learner"]["gradient_booster"]["model"]["tree_info"] == [0, 1, 2] * 4
    cfg = bst.save_config()
    assert json.loads(cfg)["learner"]["learner_model_param"]["num_target"] == "3"
    fresh = xgb.Booster()
    fresh.load_model(str(tmp_path / "m.ubj"))
    fresh.load_config(cfg)
    assert _same_bits(fresh.predict(d), p0)
    cont = xgb.train(params, d, num_boost_round=2, xgb_model=str(tmp_path / "m.json"), verbose_eval=False)
    full = xgb.train(params, d, num_boost_round=6, verbose_eval=False)
    assert _same_bits(cont.predict(d), full.predict(d))
    # another objective with num_target = 3 is refused
    doc["learner"]["objective"] = {"name": "count:poisson", "poisson_regression_param": {"max_delta_step": "0.7"}}
    bad = str(tmp_path / "bad.json")
    with open(bad, "w") as f:
        json.dump(doc, f)
    with pytest.raises(xgb.core.XGBoostError, match="num_target"):
        xgb.Booster(model_file=bad)


def test_hand_built_upstream_document(xgb, tmp_path):
    """An upstream-style document of two stumps with num_target = 2 loads and predicts (n, 2)."""
    def stump(i, thr, lo, hi):
        return {"base_weights": [0.0, lo, hi], "categories": [], "categories_nodes": [], "categories_segments": [], "categories_sizes": [],
                "default_left": [1, 0, 0], "id": i, "left_children": [1, -1, -1], "loss_changes": [1.0, 0.0, 0.0], "parents": [2147483647, 0, 0],
                "right_children": [2, -1, -1], "split_conditions": [thr, lo, hi], "split_indices": [0, 0, 0], "split_type": [0, 0, 0],
                "sum_hessian": [2.0, 1.0, 1.0], "tree_param": {"num_deleted": "0", "num_feature": "1", "num_nodes": "3", "size_leaf_vector": "1"}}
    doc = {"learner": {"attributes": {}, "feature_names": [], "feature_types": [],
                       "gradient_booster": {"model": {"gbtree_model_param": {"num_parallel_tree": "1", "num_trees": "2"}, "iteration_indptr": [0, 2],
                                                      "tree_info": [0, 1], "trees": [stump(0, 0.5, -1.0, 1.0), stump(1, 0.0, 2.0, 3.0)]}, "name": "gbtree"},
                       "learner_model_param": {"base_score": "5E-1", "boost_from_average": "1", "num_class": "0", "num_feature": "1", "num_target": "2"},
                       "objective": {"name": "reg:squarederror", "reg_loss_param": {"scale_pos_weight": "1"}}},
           "version": [3, 0, 5]}
    path = str(tmp_path / "up.json")
    with open(path, "w") as f:
        json.dump(doc, f)
    bst = xgb.Booster(model_file=path)
    X = np.array([[0.0], [1.0], [np.nan]], f32)
    np.testing.assert_array_equal(bst.predict(xgb.DMatrix(X)), np.array([[-0.5, 3.5], [1.5, 3.5], [-0.5, 2.5]], f32))


# ---------------------------------------------------------------------------------------------------------------- 7 other features
@pytest.mark.parametrize("extra", [dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7),
                                   dict(num_parallel_tree=2, subsample=0.7, colsample_bynode=0.8, seed=5),
                                   dict(colsample_bytree=0.7, colsample_bylevel=0.8, seed=6),
                                   dict(monotone_constraints="(1,0,-1,0,0,0,0,0)", interaction_constraints="[[0,1],[2,3,4]]"),
                                   dict(sampling_method="gradient_based", subsample=0.5, seed=8),
                                   dict(grow_policy="lossguide", max_depth=0, max_leaves=16)])
def test_other_features_cache_equals_predict(xgb, extra):
    X, Y = labels3(20000, 8, 101, "reg:squarederror")
    d = xgb.DMatrix(X, label=Y)
    bst = xgb.Booster(dict(BASE, objective="reg:squarederror", **extra), [d])
    for r in range(3):
        bst.update(d, r)
    P = int(extra.get("num_parallel_tree", 1))
    m = _be().booster_export_model(bst.handle)
    np.testing.assert_array_equal(m["tree_info"], np.repeat(np.arange(3), P).tolist() * 3)
    cache = _be().booster_cached_margin(bst.handle, d.handle, 3)
    pred = bst.predict(d, output_margin=True)
    if extra.get("booster") == "dart":        # predict sums fl(w_t * leaf_t) afresh; the cache carries each round's weight changes
        np.testing.assert_allclose(pred, cache, rtol=0, atol=1e-5)
    else:
        assert _same_bits(pred, cache)


# ---------------------------------------------------------------------------------------------------------------- 8 QuantileDMatrix
@pytest.mark.parametrize("objective", ["reg:squarederror", "reg:absoluteerror"])
def test_quantile_dmatrix_batches(xgb, objective):
    X, Y = labels3(9000, 6, 111, objective)

    class It(xgb.DataIter):
        def __init__(self):
            super().__init__()
            self.i = 0

        def reset(self):
            self.i = 0

        def next(self, input_data):
            if self.i == 3:
                return False
            s = slice(3000 * self.i, 3000 * (self.i + 1))
            input_data(data=X[s], label=Y[s])
            self.i += 1
            return True

    q = xgb.QuantileDMatrix(It())
    d = xgb.DMatrix(X, label=Y)
    np.testing.assert_array_equal(q.get_label(), Y.reshape(-1))
    a = xgb.train(dict(BASE, objective=objective), q, num_boost_round=3, verbose_eval=False)
    b = xgb.train(dict(BASE, objective=objective), d, num_boost_round=3, verbose_eval=False)
    assert bytes(a.save_raw("ubj")) == bytes(b.save_raw("ubj"))


# ---------------------------------------------------------------------------------------------------------------- 9 errors
def test_errors(xgb):
    X, Y = labels3(2000, 4, 121, "reg:squarederror")
    d = xgb.DMatrix(X, label=Y)
    for obj in ("count:poisson", "reg:gamma", "reg:tweedie", "binary:hinge", "multi:softprob", "reg:quantileerror", "rank:pairwise", "survival:cox"):
        with pytest.raises(xgb.core.XGBoostError, match="multi-target.*" + obj.replace(":", ".") + "|" + obj.replace(":", ".") + ".*multi-target"):
            xgb.train(dict(BASE, objective=obj, num_class=3, quantile_alpha="0.5"), d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(xgb.core.XGBoostError, match="multi_strategy"):
        xgb.train(dict(BASE, multi_strategy="multi_output_tree"), d, num_boost_round=1, verbose_eval=False)
    xgb.train(dict(BASE, multi_strategy="multi_output_tree"), xgb.DMatrix(X, label=Y[:, 0]), num_boost_round=1, verbose_eval=False)   # ignored at T = 1
    bst = xgb.train(dict(BASE), d, num_boost_round=2, verbose_eval=False)
    with pytest.raises(xgb.core.XGBoostError, match="process_type=update"):
        xgb.train(dict(BASE, process_type="update", updater="refresh"), d, num_boost_round=1, xgb_model=bst, verbose_eval=False)
    with pytest.raises(xgb.core.XGBoostError, match="base_score"):
        xgb.train(dict(BASE, base_score="[0.5, 0.5, 0.5]"), d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(xgb.core.XGBoostError, match="rows"):
        xgb.DMatrix(X, label=Y[:-1])
    with pytest.raises(xgb.core.XGBoostError, match="column"):       # a 2-column eval label against a 3-target model
        bst.eval_set([(xgb.DMatrix(X, label=Y[:, :2]), "e")])

    class Ragged(xgb.DataIter):
        def __init__(self):
            super().__init__()
            self.i = 0

        def reset(self):
            self.i = 0

        def next(self, input_data):
            if self.i == 2:
                return False
            input_data(data=X[:1000], label=Y[:1000, :2 + self.i])
            self.i += 1
            return True
    with pytest.raises(xgb.core.XGBoostError, match="columns"):
        xgb.QuantileDMatrix(Ragged())


# ---------------------------------------------------------------------------------------------------------------- 10 sklearn
def test_sklearn_regressor(xgb):
    X, Y = labels3(5000, 6, 131, "reg:squarederror")
    from sagemaker_xgboost_container_b200 import sklearn as skl
    reg = skl.XGBRegressor(n_estimators=3, max_depth=4)
    reg.fit(X, Y)
    p = reg.predict(X)
    assert p.shape == (5000, 3)
    bst = xgb.train({"objective": "reg:squarederror", "max_depth": "4", "eta": "0.3"}, xgb.DMatrix(X, label=Y), num_boost_round=3, verbose_eval=False)
    assert _same_bits(bst.predict(xgb.DMatrix(X)), p)


# ---------------------------------------------------------------------------------------------------------------- 11 two ranks
def test_two_ranks(xgb, tmp_path):
    """Two ranks train the 1-GPU model: the intercept's sums and the per-target grids are over both ranks' rows."""
    try:
        import torch
        ngpu = torch.cuda.device_count()
    except Exception:
        ngpu = 0
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    n, F, rounds = 40000, 20, 4
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29631", os.path.join(ROOT, "tests", "helpers", "multi_target_shard_worker.py"), out, str(n), str(F), str(rounds), "reg:squarederror"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, Y = labels3(n, F, 7, "reg:squarederror")
    single = xgb.train(dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256), xgb.DMatrix(X, label=Y), num_boost_round=rounds, verbose_eval=False)
    two = xgb.Booster(model_file=out)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(two.handle)
    assert m1["base_score"] == pytest.approx(m2["base_score"], rel=1e-6)
    np.testing.assert_array_equal(m1["split_index"], m2["split_index"])
