"""The forest restatement in tests/forest_reference.py against the oracle itself, the forest-aware oracle engine through the
package's Python surface (CPU), and the scikit-learn random-forest wrappers."""
import json
import pickle

import numpy as np
import pytest

import forest_reference as FR
from util import synth

TREE_KEYS = ("left", "right", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "sum_hess")


def _tree(m, t):
    a, b = int(m["tree_offset"][t]), int(m["tree_offset"][t + 1])
    return {k: np.asarray(m[k][a:b]) for k in TREE_KEYS}


def _same_tree(a, b):
    return all(np.array_equal(a[k].view(np.uint32) if a[k].dtype == np.float32 else a[k],
                              b[k].view(np.uint32) if b[k].dtype == np.float32 else b[k]) for k in TREE_KEYS)


def _params(K, **kw):
    return dict(objective="multi:softprob" if K > 1 else "reg:squarederror", num_class=K, max_depth=4, **kw)


@pytest.mark.parametrize("K", [1, 3])
def test_trees_of_a_class_are_identical_without_sampling_and_differ_with_it(oracle, K):
    X, y = synth(3000, 8, 12, "multi" if K > 1 else "reg", K=K)
    for sub, same in ((1.0, True), (0.6, False)):
        ref = FR.ForestTrainer(_params(K, eta=0.5, seed=4, subsample=sub), X, y, P=3)
        ref.update()
        m = ref.model()
        for k in range(K):
            t0 = _tree(m, 3 * k)
            for j in (1, 2):
                assert _same_tree(t0, _tree(m, 3 * k + j)) == same, (sub, k, j)


@pytest.mark.parametrize("K,colsample", [(1, 0.6), (3, 1.0)])
def test_first_tree_is_the_single_tree_with_eta_over_p(oracle, K, colsample):
    """Tree 0 of round 0 sees the rows and (at K = 1, or without column sampling) the columns of a P = 1 run; its leaves are
    fl(eta / P) times the weights, so a P = 1 run with that learning rate grows it bit for bit."""
    X, y = synth(3000, 10, 13, "multi" if K > 1 else "reg", K=K)
    P = 4
    params = _params(K, eta=0.9, subsample=0.8, colsample_bynode=colsample, seed=6, base_score=0.5)
    ref = FR.ForestTrainer(params, X, y, P=P)
    ref.update()
    single = oracle.Trainer(dict(params, eta=float(FR.forest_eta(0.9, P))), bins=ref.bins, cuts=ref.cuts, y=y, base_score=0.5)
    single.set_device_grid(X.shape[0])
    single.update()
    m, ms = ref.model(), single.model()
    for k in range(K):
        assert _same_tree(_tree(m, k * P), _tree(ms, k))
    np.testing.assert_array_equal(m["tree_info"], np.repeat(np.arange(K), P))


def test_column_sets_follow_the_position_in_the_model(oracle):
    """K = 3 with colsample_bynode: every node of the tree at position t splits on a feature of its node set drawn from
    tree_index t (split_reference.bynode_mask, the product's rule), not from the per-round numbering r * K + k."""
    from split_reference import bynode_mask
    X, y = synth(3000, 10, 14, "multi", K=3)
    ref = FR.ForestTrainer(_params(3, eta=0.7, colsample_bynode=0.3, seed=8, base_score=0.5), X, y, P=3)
    ref.update()
    m = ref.model()
    everything = np.ones(10, bool)
    for t in range(9):
        tr = _tree(m, t)
        for nid in np.nonzero(tr["left"] != -1)[0]:
            assert bynode_mask(everything, 0.3, 8, t, int(nid))[tr["split_index"][nid]], (t, nid)


@pytest.fixture
def forest_engine(monkeypatch):
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    monkeypatch.setattr(backend, "_BACKEND", FR.ForestOracleBackend(error_cls=xgb.XGBoostError))
    return xgb


@pytest.mark.parametrize("K", [1, 3])
def test_engine_layer_layout_in_model_and_config(forest_engine, K):
    xgb = forest_engine
    X, y = synth(1500, 6, 15, "multi" if K > 1 else "reg", K=K)
    params = dict(_params(K, eta=1.0, subsample=0.8, colsample_bynode=0.8, seed=1), num_parallel_tree="3")
    if K == 1:
        params.pop("num_class")
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=2)
    assert bst.num_boosted_rounds() == 2
    model = json.loads(bst.save_raw("json"))["learner"]["gradient_booster"]["model"]
    assert model["gbtree_model_param"]["num_parallel_tree"] == "3"
    assert model["iteration_indptr"] == [0, 3 * K, 6 * K]
    assert model["tree_info"] == list(np.tile(np.repeat(np.arange(K), 3), 2))
    assert json.loads(bst.save_config())["learner"]["gradient_booster"]["gbtree_model_param"]["num_parallel_tree"] == "3"
    first = bst.predict(d, output_margin=True, iteration_range=(0, 1))
    np.testing.assert_array_equal(bst[0:1].predict(d, output_margin=True), first)
    assert bst.predict(d, pred_leaf=True, iteration_range=(1, 2)).reshape(len(y), -1).shape[1] == 3 * K
    again = xgb.Booster(model_file=bst.save_raw("ubj"))
    assert again.num_boosted_rounds() == 2
    np.testing.assert_array_equal(again.predict(d, output_margin=True, iteration_range=(1, 2)),
                                  bst.predict(d, output_margin=True, iteration_range=(1, 2)))
    b3 = pickle.loads(pickle.dumps(bst))
    assert b3.num_boosted_rounds() == 2


@pytest.mark.parametrize("value", ["0", "1.5", "-2", "4abc", "abc"])
def test_engine_rejects_bad_num_parallel_tree(forest_engine, value):
    xgb = forest_engine
    X, y = synth(300, 4, 16, "reg")
    with pytest.raises(xgb.XGBoostError):
        xgb.train(dict(num_parallel_tree=value), xgb.DMatrix(X, label=y), num_boost_round=1)


def test_engine_rejects_dart_forests(forest_engine):
    xgb = forest_engine
    X, y = synth(300, 4, 17, "reg")
    with pytest.raises(xgb.XGBoostError, match="dart"):
        xgb.train(dict(booster="dart", num_parallel_tree=2), xgb.DMatrix(X, label=y), num_boost_round=1)


def test_xgbrf_fit_and_predict_on_the_engine(forest_engine):
    xgb = forest_engine
    X, y = synth(2000, 6, 18, "bin")
    clf = xgb.XGBRFClassifier(n_estimators=5, max_depth=4).fit(X, y)
    assert clf.get_booster().num_boosted_rounds() == 1
    assert len(json.loads(clf.get_booster().save_raw("json"))["learner"]["gradient_booster"]["model"]["tree_info"]) == 5
    assert (clf.predict(X) == y).mean() > max(y.mean(), 1 - y.mean())
    assert clf.predict_proba(X).shape == (2000, 2)
    Xr, yr = synth(2000, 6, 19, "reg")
    reg = xgb.XGBRFRegressor(n_estimators=4, max_depth=4).fit(Xr, yr)
    assert np.mean((reg.predict(Xr) - yr) ** 2) < np.var(yr)


def test_xgbrf_parameter_mapping(xgb):
    r = xgb.XGBRFRegressor(n_estimators=7, max_depth=3)
    p = r.get_xgb_params()
    assert p["num_parallel_tree"] == 7 and r.get_num_boosting_rounds() == 1
    assert (p["learning_rate"], p["subsample"], p["colsample_bynode"], p["reg_lambda"]) == (1.0, 0.8, 0.8, 1e-5)
    assert p["max_depth"] == 3 and "n_estimators" not in p
    c = xgb.XGBRFClassifier(n_estimators=5, subsample=0.5)
    assert c.get_xgb_params()["num_parallel_tree"] == 5 and c.get_xgb_params()["subsample"] == 0.5
    assert c.get_params()["n_estimators"] == 5
    # the plain wrappers are unchanged
    assert "num_parallel_tree" not in xgb.XGBRegressor(n_estimators=7).get_xgb_params()
    assert xgb.XGBRegressor(n_estimators=7).get_num_boosting_rounds() == 7
    X, y = synth(100, 3, 20, "reg")
    with pytest.raises(NotImplementedError):
        xgb.XGBRFRegressor(early_stopping_rounds=2).fit(X, y)
    with pytest.raises(NotImplementedError):
        xgb.XGBRFRegressor(callbacks=[object()]).fit(X, y)


def test_num_parallel_tree_is_forwarded(xgb):
    from sagemaker_xgboost_container_b200.core import _DROP, _check_unapplied
    assert _check_unapplied("num_parallel_tree", "4") == "4"
    assert _check_unapplied("num_parallel_tree", 1) is not _DROP
