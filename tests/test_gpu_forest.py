"""Boosted random forests (num_parallel_tree = P > 1) on the GPU: trees against the forest restatement in
tests/forest_reference.py, layer-indexed prediction, slicing and SHAP, model IO of the layer layout, graph replay and the
container's string hyperparameters."""
import json
import pickle

import numpy as np
import pytest

import forest_reference as FR
from test_gpu_tree_graph import _train_in_subprocess
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ARRAYS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")
LEAF_TOL = 1e-5
MARGIN_TOL = 2e-5


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _forest(xgb, X, y, params, rounds):
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    for r in range(rounds):
        bst.update(d, r)
    return d, bst


PARITY = {
    # name: (objective, kind, K, P, extra params, bit exact)
    "squarederror-P3": ("reg:squarederror", "reg", 1, 3, dict(subsample=0.8, colsample_bynode=0.8), True),
    "hinge-P4": ("binary:hinge", "bin", 1, 4, dict(subsample=0.8, colsample_bynode=0.8), True),
    "logistic-P4": ("binary:logistic", "bin", 1, 4, dict(subsample=0.8, colsample_bynode=0.8), False),
    "softprob-K3-P3": ("multi:softprob", "multi", 3, 3, dict(subsample=0.8, colsample_bynode=0.8), False),
    "softprob-K3-P3-rows": ("multi:softprob", "multi", 3, 3, dict(subsample=0.8), False),
    "lossguide-P3": ("reg:squarederror", "reg", 1, 3, dict(subsample=0.8, grow_policy="lossguide", max_leaves=12, max_depth=0), True),
}


@pytest.mark.parametrize("case", sorted(PARITY))
def test_trees_match_the_forest_reference(xgb, oracle, case):
    objective, kind, K, P, extra, exact = PARITY[case]
    X, y = synth(12000, 16, 21, kind, K=K)
    params = dict(objective=objective, tree_method="hist", max_bin=256, max_depth=5, eta=0.7, base_score=0.5, seed=5, num_parallel_tree=P)
    params.update(extra)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    ref = FR.ForestTrainer(params, X, y, P, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256),
                           base_score=0.5)
    rounds = 3
    for r in range(rounds):
        bst.update(d, r)
        ref.update()
    assert bst.num_boosted_rounds() == rounds
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    np.testing.assert_array_equal(m["tree_info"], np.tile(np.repeat(np.arange(K), P), rounds))
    cache = _be().booster_cached_margin(bst.handle, d.handle, K)
    margin = bst.predict(d, output_margin=True).reshape(-1, K)
    if exact:
        for k in ARRAYS:
            a, b = (m[k], mr[k]) if m[k].dtype != np.float32 else (_u32(m[k]), _u32(mr[k]))
            np.testing.assert_array_equal(a, b, err_msg=k)
        np.testing.assert_array_equal(_u32(cache), _u32(ref.margins()))
        np.testing.assert_array_equal(_u32(margin), _u32(ref.margins()))
    else:
        assert max_leaf_diff(m, mr) <= LEAF_TOL
        np.testing.assert_allclose(cache, ref.margins(), rtol=0, atol=MARGIN_TOL)
        np.testing.assert_allclose(margin, ref.margins(), rtol=0, atol=MARGIN_TOL)
    # the P trees of a class are different trees (each has its own rows)
    t = m["tree_offset"]
    assert any(not np.array_equal(m["split_index"][t[0]:t[1]], m["split_index"][t[j]:t[j + 1]]) or t[1] - t[0] != t[j + 1] - t[j]
               for j in range(1, P))


def test_first_tree_equals_a_single_tree_and_no_sampling_gives_equal_trees(xgb):
    X, y = synth(20000, 20, 22, "multi", K=3)
    base = dict(objective="multi:softprob", num_class=3, tree_method="hist", max_depth=5, eta=0.8, base_score=0.5, seed=9)
    _, forest = _forest(xgb, X, y, dict(base, num_parallel_tree=4, subsample=0.7), 1)
    _, single = _forest(xgb, X, y, dict(base, eta=float(FR.forest_eta(0.8, 4)), subsample=0.7), 1)
    mf, ms = _be().booster_export_model(forest.handle), _be().booster_export_model(single.handle)
    for k in range(3):
        a0, a1 = mf["tree_offset"][4 * k], mf["tree_offset"][4 * k + 1]
        b0, b1 = ms["tree_offset"][k], ms["tree_offset"][k + 1]
        for key in ARRAYS:
            np.testing.assert_array_equal(mf[key][a0:a1], ms[key][b0:b1], err_msg="class %d %s" % (k, key))
    _, same = _forest(xgb, X, y, dict(base, num_parallel_tree=3), 2)
    m = _be().booster_export_model(same.handle)
    to = m["tree_offset"]
    for t in range(m["tree_info"].size):
        if t % 3:
            np.testing.assert_array_equal(_u32(m["split_cond"][to[t]:to[t + 1]]), _u32(m["split_cond"][to[t - t % 3]:to[t - t % 3 + 1]]))


@pytest.fixture(scope="module")
def small_forest(xgb):
    X, y = synth(4000, 6, 23, "multi", K=3)
    params = dict(objective="multi:softprob", num_class=3, tree_method="hist", max_depth=4, eta=0.5, seed=1, subsample=0.8,
                  colsample_bynode=0.8, num_parallel_tree=3)
    d, bst = _forest(xgb, X, y, params, 5)
    return X, y, d, bst


def test_layer_indexed_prediction(xgb, oracle, small_forest):
    X, y, d, bst = small_forest
    K, P = 3, 3
    m = dict(_be().booster_export_model(bst.handle), objective="multi:softprob")
    assert bst.num_boosted_rounds() == 5 and m["tree_info"].size == 5 * K * P
    for a, b in ((0, 1), (1, 3), (2, 5), (0, 5)):
        got = bst.predict(d, output_margin=True, iteration_range=(a, b))
        want = oracle.predict_margin(m, X, a * K * P, b * K * P)
        np.testing.assert_array_equal(_u32(got), _u32(want))
        leaf = bst.predict(d, pred_leaf=True, iteration_range=(a, b))
        np.testing.assert_array_equal(leaf.reshape(X.shape[0], -1), oracle.predict_leaf(m, X, a * K * P, b * K * P))
        sl = bst[a:b]
        assert sl.num_boosted_rounds() == b - a
        np.testing.assert_array_equal(_u32(sl.predict(d, output_margin=True)), _u32(got))
        contribs = bst.predict(d, pred_contribs=True, iteration_range=(a, b))
        np.testing.assert_allclose(contribs.sum(axis=-1), got, rtol=0, atol=1e-4)
    shap = bst.predict(d, pred_contribs=True, iteration_range=(1, 3))[:64]
    np.testing.assert_allclose(shap, oracle.shap_bruteforce(m, X[:64], K * P, 3 * K * P), rtol=0, atol=1e-4)
    with pytest.raises(xgb.core.XGBoostError):
        bst.predict(d, iteration_range=(0, 6))


def test_model_io_round_trips(xgb, small_forest, tmp_path):
    X, y, d, bst = small_forest
    want = bst.predict(d, output_margin=True, iteration_range=(1, 4))
    doc = json.loads(bst.save_raw("json"))
    gb = doc["learner"]["gradient_booster"]["model"]
    assert gb["gbtree_model_param"]["num_parallel_tree"] == "3"
    assert list(gb["iteration_indptr"]) == [9 * r for r in range(6)]
    assert json.loads(bst.save_config())["learner"]["gradient_booster"]["gbtree_model_param"]["num_parallel_tree"] == "3"
    for raw in (bst.save_raw("json"), bst.save_raw("ubj")):
        b2 = xgb.Booster(model_file=bytearray(raw))
        assert b2.num_boosted_rounds() == 5
        np.testing.assert_array_equal(_u32(b2.predict(d, output_margin=True, iteration_range=(1, 4))), _u32(want))
    b3 = pickle.loads(pickle.dumps(bst))
    assert b3.num_boosted_rounds() == 5
    np.testing.assert_array_equal(_u32(b3.predict(d, output_margin=True, iteration_range=(1, 4))), _u32(want))


def test_pickled_forest_trains_on_as_a_forest(xgb):
    X, y = synth(15000, 12, 24, "reg")
    params = dict(objective="reg:squarederror", tree_method="hist", max_depth=5, eta=1.0, seed=2, subsample=0.8, colsample_bynode=0.8,
                  num_parallel_tree=4)
    d, whole = _forest(xgb, X, y, params, 3)
    d2, part = _forest(xgb, X, y, params, 2)
    resumed = pickle.loads(pickle.dumps(part))
    resumed.update(d2, 2)
    mw, mr = _be().booster_export_model(whole.handle), _be().booster_export_model(resumed.handle)
    for k in ARRAYS:
        if k != "split_bin":            # a loaded model keeps thresholds, not bin ids: compare those of the new round only
            np.testing.assert_array_equal(mw[k], mr[k], err_msg=k)
    new = slice(int(mw["tree_offset"][8]), None)
    np.testing.assert_array_equal(mw["split_bin"][new], mr["split_bin"][new])
    assert resumed.num_boosted_rounds() == 3


def test_single_class_layout_in_model_and_config(xgb):
    X, y = synth(3000, 8, 28, "reg")
    _, bst = _forest(xgb, X, y, dict(objective="reg:squarederror", max_depth=4, subsample=0.8, num_parallel_tree=4), 3)
    model = json.loads(bst.save_raw("json"))["learner"]["gradient_booster"]["model"]
    assert model["gbtree_model_param"]["num_parallel_tree"] == "4"
    assert list(model["iteration_indptr"]) == [0, 4, 8, 12] and list(model["tree_info"]) == [0] * 12
    assert json.loads(bst.save_config())["learner"]["gradient_booster"]["gbtree_model_param"]["num_parallel_tree"] == "4"
    assert bst.num_boosted_rounds() == 3 and bst[1:3].num_boosted_rounds() == 2


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_rank_forest_equals_single_gpu(xgb, tmp_path):
    """P = 3 with column sampling and no row sampling, rows sharded over 2 ranks: the same model as one GPU, bit for bit."""
    import os
    import subprocess
    import sys
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n, F, rounds = 40000, 20, 3
    extra = dict(num_parallel_tree=3, colsample_bynode=0.8, seed=5)
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29613", os.path.join(root, "tests", "helpers", "train_shard_worker.py"), out, str(n), str(F), str(rounds), "reg:squarederror", repr(extra)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y = synth(n, F, 7, "reg")
    single = xgb.train(dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256, **extra), xgb.DMatrix(X, label=y),
                       num_boost_round=rounds, verbose_eval=False)
    multi = xgb.Booster(model_file=out)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(multi.handle)
    assert_same_structure(m2, m1)
    np.testing.assert_array_equal(_u32(m2["split_cond"]), _u32(m1["split_cond"]))
    assert multi.num_boosted_rounds() == rounds


def _doc_without(raw, drop_indptr=False, **model_edits):
    doc = json.loads(raw)
    model = doc["learner"]["gradient_booster"]["model"]
    if drop_indptr:
        del model["iteration_indptr"]
    model.update(model_edits)
    return bytearray(json.dumps(doc).encode())


def test_hand_built_documents(xgb, small_forest):
    X, y, d, bst = small_forest
    raw = bst.save_raw("json")
    want = bst.predict(d, output_margin=True, iteration_range=(2, 4))
    for buf in (_doc_without(raw), _doc_without(raw, drop_indptr=True)):     # with iteration_indptr, and 1.x style without it
        b = xgb.Booster(model_file=buf)
        assert b.num_boosted_rounds() == 5
        np.testing.assert_array_equal(_u32(b.predict(d, output_margin=True, iteration_range=(2, 4))), _u32(want))
    bad = [dict(iteration_indptr=[1] + [9 * r for r in range(1, 6)]),
           dict(iteration_indptr=[0, 9, 5, 27, 36, 45]),
           dict(iteration_indptr=[0, 9, 18, 27, 36]),
           dict(iteration_indptr=[0, 9, 18, 27, 36, 46]),
           dict(iteration_indptr=[]),
           dict(iteration_indptr=[0, 4.5, 18, 27, 36, 45])]
    for edit in bad:
        with pytest.raises(xgb.core.XGBoostError):
            xgb.Booster(model_file=_doc_without(raw, **edit))
    with pytest.raises(xgb.core.XGBoostError):        # without iteration_indptr, 45 trees are not whole rounds of 3 x 4
        xgb.Booster(model_file=_doc_without(raw, drop_indptr=True, gbtree_model_param={"num_parallel_tree": "4", "num_trees": "45"}))


@pytest.mark.parametrize("value", ["0", "1.5", "-2", "abc", "4abc", "3x"])
def test_bad_num_parallel_tree_is_rejected(xgb, value):
    X, y = synth(500, 4, 25, "reg")
    with pytest.raises(xgb.core.XGBoostError):
        xgb.train(dict(num_parallel_tree=value), xgb.DMatrix(X, label=y), num_boost_round=1)


def test_dart_forest_is_rejected_for_training_and_served(xgb):
    X, y = synth(500, 4, 26, "reg")
    d = xgb.DMatrix(X, label=y)
    with pytest.raises(xgb.core.XGBoostError, match="dart"):
        xgb.train(dict(booster="dart", num_parallel_tree=2), d, num_boost_round=1)
    # a dart model written with two trees per round (as xgboost writes dart forests) loads and predicts by round
    bst = xgb.train(dict(booster="dart", rate_drop=0.3, one_drop=1, max_depth=3, seed=2), d, num_boost_round=6)
    doc = json.loads(bst.save_raw("json"))
    model = doc["learner"]["gradient_booster"]["gbtree"]["model"]
    model["gbtree_model_param"]["num_parallel_tree"] = "2"
    model["iteration_indptr"] = [0, 2, 4, 6]
    forest = xgb.Booster(model_file=bytearray(json.dumps(doc).encode()))
    assert forest.num_boosted_rounds() == 3
    np.testing.assert_array_equal(_u32(forest.predict(d, output_margin=True)), _u32(bst.predict(d, output_margin=True)))
    np.testing.assert_array_equal(_u32(forest.predict(d, output_margin=True, iteration_range=(1, 2))),
                                  _u32(bst.predict(d, output_margin=True, iteration_range=(2, 4))))


def test_container_string_hyperparameters(xgb):
    X, y = synth(20000, 10, 27, "bin")
    hp = {"objective": "binary:logistic", "num_parallel_tree": "4", "eta": "1", "subsample": "0.8", "colsample_bynode": "0.8",
          "max_depth": "5"}
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(hp, d, num_boost_round=2)
    assert bst.num_boosted_rounds() == 2
    cfg = json.loads(bst.save_config())
    assert cfg["learner"]["gradient_booster"]["gbtree_model_param"]["num_parallel_tree"] == "4"
    full = bst.predict(d)
    first = bst.predict(d, iteration_range=(0, 1))         # what serving does with best_ntree_limit = 1
    assert full.shape == first.shape == (X.shape[0],) and not np.array_equal(full, first)
    rf = xgb.XGBRFClassifier(n_estimators=6, max_depth=4).fit(X, y)
    assert rf.get_booster().num_boosted_rounds() == 1
    assert _be().booster_export_model(rf.get_booster().handle)["tree_info"].size == 6
    assert (rf.predict(X) == y).mean() > max(y.mean(), 1 - y.mean())      # better than the majority class


GRAPH_CASES = {
    "squarederror-rows-columns": dict(params=dict(tree_method="hist", max_bin=256, eta=1.0, max_depth=6, objective="reg:squarederror",
                                                  num_parallel_tree=4, subsample=0.8, colsample_bynode=0.8, seed=3),
                                      rounds=3, data=[[60000, 40, 3, "reg", 1]]),
    "softprob-columns-only": dict(params=dict(tree_method="hist", max_bin=256, eta=1.0, max_depth=5, objective="multi:softprob", num_class=3,
                                              num_parallel_tree=3, colsample_bynode=0.7, seed=4),
                                  rounds=2, data=[[50000, 30, 7, "multi", 3]]),
}


@pytest.mark.parametrize("case", sorted(GRAPH_CASES))
def test_forest_graph_replay_equals_direct_issue(tmp_path, case):
    cfg = GRAPH_CASES[case]
    replayed = _train_in_subprocess(tmp_path, cfg, False)
    direct = _train_in_subprocess(tmp_path, cfg, True)
    assert replayed.keys() == direct.keys()
    for k in replayed:
        np.testing.assert_array_equal(replayed[k], direct[k], err_msg=k)
