"""rank:pairwise, rank:ndcg and rank:map on the GPU: gradients against tests/ranking_reference.py through
XGB200BoosterComputeGradient, their determinism, the ndcg / map metrics, query groups on the DMatrix (group, qid, group_ptr,
slicing, the libsvm qid routes), training, model IO and serving, XGBRanker, and the errors."""
import ctypes as C
import json
import os
import pickle

import numpy as np
import pytest

import ranking_reference as RR
from util import synth

pytestmark = pytest.mark.gpu
OBJECTIVES = ["rank:pairwise", "rank:ndcg", "rank:map"]


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _ptr(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def _labels(objective, n, rng, levels=5):
    if objective == "rank:map":
        return (rng.random(n) < 0.3).astype(np.float32)
    return rng.integers(0, levels, n).astype(np.float32)


def _check_gradient(xgb, objective, sizes, seed, weighted=False, params=None, margin=None, labels=None):
    rng = np.random.default_rng(seed)
    ptr = _ptr(sizes)
    n = int(ptr[-1])
    X = rng.standard_normal((n, 3)).astype(np.float32)
    y = _labels(objective, n, rng) if labels is None else labels
    w = rng.uniform(0.2, 3.0, len(sizes)).astype(np.float32) if weighted else None
    d = xgb.DMatrix(X, label=y, weight=w, group=sizes)
    p = dict(objective=objective, **(params or {}))
    bst = xgb.Booster(p, [d])
    m = (rng.standard_normal(n) * 2).astype(np.float32) if margin is None else margin
    got = _be().booster_compute_gradient(bst.handle, d.handle, m)[:, 0, :]
    mean = p.get("lambdarank_pair_method") == "mean"
    ref_kw = dict(k=int(p.get("lambdarank_num_pair_per_sample", 1 if mean else 32)), mean=mean, seed=int(p.get("seed", 0)), exp_gain=p.get("ndcg_exp_gain", True) in (True, 1, "1", "true"),
                  normalization=p.get("lambdarank_normalization", True) in (True, 1, "1", "true"),
                  score_normalization=p.get("lambdarank_score_normalization", True) in (True, 1, "1", "true"))
    want = RR.gradient(m, y, ptr, w, objective, **ref_kw)
    assert np.all(np.isfinite(got)) and np.all(got[:, 1] >= 0)
    u = _ulps(got, want).max(axis=1)
    # the device sums each document's pairs in a different (fixed) order than the restatement: double rounding that reaches the
    # float result rarely, and then by one ulp
    assert (u <= 2).mean() >= 0.999, (objective, int((u > 2).sum()), float(np.abs(got - want).max()))
    assert np.abs(got - want).max() <= 1e-6 * max(1.0, float(np.abs(want).max())), (objective, float(np.abs(got - want).max()))
    return d, bst, m, got


@pytest.mark.parametrize("objective", OBJECTIVES)
@pytest.mark.parametrize("norm", [(True, True), (False, False), (True, False), (False, True)])
@pytest.mark.parametrize("weighted", [False, True])
def test_gradient_matches_reference(xgb, objective, norm, weighted):
    rng = np.random.default_rng(7)
    sizes = rng.integers(1, 120, 300)
    _check_gradient(xgb, objective, sizes, 11, weighted, dict(lambdarank_normalization=norm[0], lambdarank_score_normalization=norm[1]))


@pytest.mark.parametrize("objective", OBJECTIVES)
def test_gradient_group_mixes(xgb, objective):
    _check_gradient(xgb, objective, np.ones(5000, np.int64), 1)                        # no pairs at all
    _check_gradient(xgb, objective, np.full(20000, 2), 2)
    _check_gradient(xgb, objective, np.full(100000, 3), 3, weighted=True)
    _check_gradient(xgb, objective, np.array([200000]), 4, params=dict(lambdarank_num_pair_per_sample=8))
    n = 3000
    rng = np.random.default_rng(5)
    _check_gradient(xgb, objective, np.array([1000, 2000]), 5, margin=np.zeros(n, np.float32))    # all equal: no score normalization
    heavy = (rng.random(n) < 0.05).astype(np.float32)                                                 # heavy label ties
    _check_gradient(xgb, objective, np.array([n]), 6, labels=heavy, params=dict(lambdarank_num_pair_per_sample=100))


@pytest.mark.parametrize("objective", OBJECTIVES)
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("weighted", [False, True])
def test_mean_pairs_match_reference(xgb, objective, k, weighted):
    """lambdarank_pair_method=mean: the draws, the pair terms and their fixed-point sums against the restatement."""
    rng = np.random.default_rng(21)
    sizes = rng.integers(1, 80, 300)
    for norm in ((True, True), (False, False)):
        _check_gradient(xgb, objective, sizes, 22, weighted, dict(lambdarank_pair_method="mean", lambdarank_num_pair_per_sample=k, seed=5,
                                                                  lambdarank_normalization=norm[0], lambdarank_score_normalization=norm[1]))
    _check_gradient(xgb, objective, np.array([30000]), 23, params=dict(lambdarank_pair_method="mean", lambdarank_num_pair_per_sample=k))


def test_mean_pairs_deterministic(xgb):
    rng = np.random.default_rng(24)
    sizes = rng.integers(1, 500, 3000)
    n = int(sizes.sum())
    X = rng.standard_normal((n, 2)).astype(np.float32)
    d = xgb.DMatrix(X, label=rng.integers(0, 5, n).astype(np.float32), group=sizes)
    bst = xgb.Booster({"objective": "rank:ndcg", "lambdarank_pair_method": "mean", "lambdarank_num_pair_per_sample": 4}, [d])
    m = rng.standard_normal(n).astype(np.float32)
    runs = [_be().booster_compute_gradient(bst.handle, d.handle, m) for _ in range(3)]
    for r in runs[1:]:
        np.testing.assert_array_equal(r.view(np.uint32), runs[0].view(np.uint32))
    other_round = _be().booster_compute_gradient(bst.handle, d.handle, m, round=1)
    assert not np.array_equal(other_round, runs[0])            # each round draws its own partners


def test_gradient_without_groups_is_one_group(xgb):
    rng = np.random.default_rng(8)
    n = 500
    X = rng.standard_normal((n, 2)).astype(np.float32)
    y = rng.integers(0, 3, n).astype(np.float32)
    m = rng.standard_normal(n).astype(np.float32)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster({"objective": "rank:ndcg"}, [d])
    got = _be().booster_compute_gradient(bst.handle, d.handle, m)[:, 0, :]
    assert (_ulps(got, RR.gradient(m, y, None)).max(axis=1) <= 2).all()


@pytest.mark.parametrize("objective", OBJECTIVES)
def test_gradient_deterministic_and_independent_of_group_order(xgb, objective):
    rng = np.random.default_rng(9)
    sizes = rng.integers(1, 300, 2000)
    ptr = _ptr(sizes)
    n = int(ptr[-1])
    X = rng.standard_normal((n, 3)).astype(np.float32)
    y = _labels(objective, n, rng)
    m = rng.standard_normal(n).astype(np.float32)
    w = rng.uniform(0.5, 2, len(sizes)).astype(np.float32)
    d = xgb.DMatrix(X, label=y, weight=w, group=sizes)
    bst = xgb.Booster({"objective": objective}, [d])
    runs = [_be().booster_compute_gradient(bst.handle, d.handle, m) for _ in range(3)]
    for r in runs[1:]:
        np.testing.assert_array_equal(r.view(np.uint32), runs[0].view(np.uint32))
    perm_groups = rng.permutation(len(sizes))
    rows = np.concatenate([np.arange(ptr[g], ptr[g + 1]) for g in perm_groups])
    d2 = xgb.DMatrix(X[rows], label=y[rows], weight=w[perm_groups], group=sizes[perm_groups])
    bst2 = xgb.Booster({"objective": objective}, [d2])
    got = _be().booster_compute_gradient(bst2.handle, d2.handle, m[rows])
    np.testing.assert_array_equal(got.view(np.uint32), runs[0][rows].view(np.uint32))


@pytest.mark.parametrize("weighted", [False, True])
def test_metrics_match_reference(xgb, weighted):
    rng = np.random.default_rng(10)
    mats = []
    for seed in (0, 1):
        sizes = rng.integers(1, 60, 400)
        n = int(sizes.sum())
        X = rng.standard_normal((n, 4)).astype(np.float32)
        y = rng.integers(0, 4, n).astype(np.float32)
        y[rng.random(n) < 0.3] = 0
        w = rng.uniform(0.2, 3, len(sizes)).astype(np.float32) if weighted else None
        mats.append((xgb.DMatrix(X, label=y, weight=w, group=sizes), y, _ptr(sizes), w))
    names = ["ndcg", "ndcg@3", "ndcg-", "ndcg@5-", "map", "map@3", "map-", "map@10-"]
    bst = xgb.train({"objective": "rank:ndcg", "eval_metric": names, "max_depth": 3}, mats[0][0], 3)
    res = bst.eval_set([(mats[0][0], "train"), (mats[1][0], "eval")])
    got = {tok.split(":")[0]: float(tok.split(":")[1]) for tok in res.split("\t")[1:]}
    for (dm, y, ptr, w), tag in zip(mats, ("train", "eval")):
        m = bst.predict(dm, output_margin=True)
        for name in names:
            want = RR.metric(m, y, ptr, w, name, exp_gain=True)
            assert got["%s-%s" % (tag, name)] == pytest.approx(want, rel=1e-12, abs=1e-14), (tag, name)


def _rank_data(rng, G=300, F=6):
    sizes = rng.integers(2, 40, G)
    n = int(sizes.sum())
    X, _ = synth(n, F, int(rng.integers(0, 1000)), "reg")
    score = X[:, 0] + 0.5 * X[:, 1] + 0.3 * rng.standard_normal(n)
    y = np.clip(np.round(score + 1.5), 0, 4).astype(np.float32)
    return X, y, sizes


@pytest.mark.parametrize("objective", OBJECTIVES)
def test_training_improves_the_default_metric(xgb, objective):
    rng = np.random.default_rng(12)
    X, y, sizes = _rank_data(rng)
    if objective == "rank:map":
        y = (y >= 3).astype(np.float32)
    d = xgb.DMatrix(X, label=y, group=sizes)
    res = {}
    xgb.train({"objective": objective, "max_depth": 4}, d, 20, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    (name, vals), = res["train"].items()
    assert name == ("map@32" if objective == "rank:map" else "ndcg@32")
    assert vals[-1] > vals[0]
    res = {}
    xgb.train({"objective": objective, "max_depth": 4, "lambdarank_pair_method": "mean"}, d, 20, evals=[(d, "train")], evals_result=res,
              verbose_eval=False)
    (name, vals), = res["train"].items()
    assert name == ("map" if objective == "rank:map" else "ndcg")
    assert vals[-1] > vals[0]


@pytest.mark.parametrize("objective,mean", [("rank:ndcg", False), ("rank:map", False), ("rank:pairwise", True)])
def test_trees_match_oracle_fed_the_same_pairs(xgb, objective, mean):
    """Trees grown from the device gradients equal the oracle trainer's trees grown from the same pairs (carrier labels)."""
    import survival_reference as SR
    from oracle import gbt_oracle as O
    from util import assert_same_structure, max_leaf_diff
    rng = np.random.default_rng(25)
    X, y, sizes = _rank_data(rng, G=400, F=8)
    if objective == "rank:map":
        y = (y >= 3).astype(np.float32)
    n = len(y)
    w = rng.uniform(0.5, 2.0, len(sizes)).astype(np.float32)
    d = xgb.DMatrix(X, label=y, weight=w, group=sizes)
    params = dict(objective=objective, tree_method="hist", max_bin=256, max_depth=5, eta=0.5, seed=3)
    if mean:
        params.update(lambdarank_pair_method="mean", lambdarank_num_pair_per_sample=2)
    bst = xgb.Booster(params, [d])
    probe = xgb.Booster(params, [d])
    op = dict(tree_method="hist", max_bin=256, max_depth=5, eta=0.5, objective="reg:squarederror", base_score=0.5)
    t = O.Trainer(op, X=X, y=np.zeros(n, np.float32), weights=np.ones(n, np.float32), bins=_be().dmatrix_get_bins(d.handle, 256),
                  cuts=_be().dmatrix_get_cuts(d.handle, 256), base_score=0.5)
    t.set_device_grid()
    m = np.full(n, 0.5, np.float32)
    for r in range(3):
        gp = _be().booster_compute_gradient(probe.handle, d.handle, m, round=r)[:, 0, :]
        t.y[:], t.w[:] = SR.carrier(gp)
        t.set_margins(np.zeros(n, np.float32))
        t.update()
        m = (m + t.margins()[:, 0]).astype(np.float32)
        bst.update(d, r)
    mg, mr = _be().booster_export_model(bst.handle), t.model()
    assert_same_structure(mg, mr)
    assert max_leaf_diff(mg, mr) <= 1e-5


def test_group_info_round_trips(xgb):
    X = np.zeros((10, 2), np.float32)
    d = xgb.DMatrix(X, label=np.zeros(10))
    assert len(d.get_group()) == 0 and len(d.get_uint_info("group_ptr")) == 0
    d.set_group([3, 0, 7])
    np.testing.assert_array_equal(d.get_uint_info("group_ptr"), [0, 3, 3, 10])
    np.testing.assert_array_equal(d.get_group(), [3, 0, 7])
    d.set_uint_info("group_ptr", [0, 4, 10])
    np.testing.assert_array_equal(d.get_group(), [4, 6])
    d.set_info(qid=np.array([1, 1, 2, 2, 2, 5, 5, 5, 5, 9]))
    np.testing.assert_array_equal(d.get_uint_info("group_ptr"), [0, 2, 5, 9, 10])
    np.testing.assert_array_equal(xgb.DMatrix(X, qid=[0] * 4 + [3] * 6).get_group(), [4, 6])
    with pytest.raises(xgb.XGBoostError, match="non-decreasing"):
        d.set_info(qid=[1, 2, 1, 3, 3, 3, 3, 3, 3, 3])
    with pytest.raises(xgb.XGBoostError, match="add up to num_row"):
        d.set_group([3, 3])
    with pytest.raises(xgb.XGBoostError, match="group_ptr must not decrease"):
        d.set_uint_info("group_ptr", [0, 5, 4, 10])


def test_slice_by_whole_groups(xgb):
    rng = np.random.default_rng(13)
    X = rng.standard_normal((10, 2)).astype(np.float32)
    d = xgb.DMatrix(X, label=np.arange(10), weight=[1, 2, 3], group=[3, 3, 4])
    with pytest.raises(xgb.XGBoostError, match="allow_groups=True"):
        d.slice([0, 1, 2])
    with pytest.raises(xgb.XGBoostError, match="whole query groups"):
        d.slice([0, 1], allow_groups=True)
    s = d.slice([6, 7, 8, 9, 0, 1, 2], allow_groups=True)
    np.testing.assert_array_equal(s.get_group(), [4, 3])
    np.testing.assert_array_equal(s.get_weight(), [3, 1])
    np.testing.assert_array_equal(s.get_label(), [6, 7, 8, 9, 0, 1, 2])


def _write_qid_dir(path, rng, groups=60):
    os.makedirs(path, exist_ok=True)
    lines, q = [], 0
    for g in range(groups):
        q += int(rng.integers(1, 3))
        for _ in range(int(rng.integers(2, 25))):
            x = rng.standard_normal(5)
            rel = int(np.clip(np.round(x[0] + x[1] + 1.5), 0, 4))
            lines.append("%d qid:%d " % (rel, q) + " ".join("%d:%.5g" % (i, v) for i, v in enumerate(x)))
    half = len(lines) // 2
    for k, chunk in enumerate((lines[:half], lines[half:])):      # a group may continue into the next file
        with open(os.path.join(path, "part-%d" % k), "w") as fh:
            fh.write("\n".join(chunk) + "\n")


def test_libsvm_qid_channel_end_to_end(xgb, tmp_path):
    rng = np.random.default_rng(14)
    path = str(tmp_path / "train")
    _write_qid_dir(path, rng)
    d = xgb.DMatrix(path + "?format=libsvm")
    assert len(d.get_group()) > 1 and int(d.get_group().sum()) == d.num_row()
    be = _be()
    h = C.c_void_p()
    be._check(be.lib.XGDMatrixCreateFromURI(C.c_char_p(json.dumps({"uri": path + "?format=libsvm"}).encode()), C.byref(h)))
    d2 = xgb.DMatrix._from_handle(h)
    np.testing.assert_array_equal(d2.get_uint_info("group_ptr"), d.get_uint_info("group_ptr"))
    np.testing.assert_array_equal(d2.get_label(), d.get_label())
    res = {}
    # the container's string hyperparameters
    params = {"objective": "rank:ndcg", "eval_metric": "ndcg@5", "max_depth": "4", "eta": "0.3", "lambdarank_pair_method": "topk",
              "lambdarank_num_pair_per_sample": "8", "ndcg_exp_gain": "true", "lambdarank_normalization": "false"}
    xgb.train(params, d2, 20, evals=[(d2, "train")], evals_result=res, verbose_eval=False)
    v = res["train"]["ndcg@5"]
    assert v[-1] > v[0]


def test_model_io_serving_and_resume(xgb, tmp_path):
    rng = np.random.default_rng(15)
    X, y, sizes = _rank_data(rng)
    d = xgb.DMatrix(X, label=y, group=sizes)
    params = {"objective": "rank:pairwise", "max_depth": 3, "lambdarank_num_pair_per_sample": 5, "ndcg_exp_gain": False}
    bst = xgb.train(params, d, 6)
    pred = bst.predict(d)
    np.testing.assert_array_equal(pred, bst.predict(d, output_margin=True))
    lp = json.loads(bst.save_config())["learner"]["objective"]["lambdarank_param"]
    assert lp["lambdarank_num_pair_per_sample"] == "5" and lp["ndcg_exp_gain"] == "0" and lp["lambdarank_pair_method"] == "topk"
    for fmt in ("json", "ubj"):
        f = str(tmp_path / ("m." + fmt))
        bst.save_model(f)
        b2 = xgb.Booster(model_file=f)
        np.testing.assert_array_equal(b2.predict(d), pred)
        assert json.loads(b2.save_config())["learner"]["objective"]["lambdarank_param"] == lp
    b3 = pickle.loads(pickle.dumps(bst))
    np.testing.assert_array_equal(b3.predict(d), pred)
    np.testing.assert_array_equal(bst[0:3].predict(d), xgb.train(params, d, 3).predict(d))
    # resume: 3 + 3 rounds from a saved model give the 6-round model
    f = str(tmp_path / "m3.json")
    xgb.train(params, d, 3).save_model(f)
    resumed = xgb.train(params, d, 3, xgb_model=f)
    np.testing.assert_array_equal(resumed.predict(d), pred)
    from sagemaker_xgboost_container_b200 import serving
    out = serving.predict(bst, "json", d, "text/libsvm", objective="rank:pairwise")
    np.testing.assert_array_equal(np.asarray(out, np.float32), pred)


def test_upstream_shaped_document_loads(xgb):
    """A ranking document shaped like upstream's: lambdarank_param with only some fields, values as strings."""
    X = np.array([[0.0], [1.0]], np.float32)
    doc = {"learner": {"attributes": {}, "feature_names": [], "feature_types": [],
                       "gradient_booster": {"model": {"gbtree_model_param": {"num_parallel_tree": "1", "num_trees": "1"}, "iteration_indptr": [0, 1],
                                                      "tree_info": [0], "trees": [{
                                                          "base_weights": [0.0, -0.25, 0.5], "categories": [], "categories_nodes": [],
                                                          "categories_segments": [], "categories_sizes": [], "default_left": [1, 0, 0], "id": 0,
                                                          "left_children": [1, -1, -1], "loss_changes": [1.0, 0.0, 0.0], "parents": [2147483647, 0, 0],
                                                          "right_children": [2, -1, -1], "split_conditions": [0.5, -0.25, 0.5],
                                                          "split_indices": [0, 0, 0], "split_type": [0, 0, 0], "sum_hessian": [2.0, 1.0, 1.0],
                                                          "tree_param": {"num_deleted": "0", "num_feature": "1", "num_nodes": "3", "size_leaf_vector": "1"}}]},
                                              "name": "gbtree"},
                       "learner_model_param": {"base_score": "5E-1", "boost_from_average": "1", "num_class": "0", "num_feature": "1", "num_target": "1"},
                       "objective": {"name": "rank:ndcg", "lambdarank_param": {"lambdarank_num_pair_per_sample": "4", "lambdarank_pair_method": "mean"}}},
           "version": [3, 0, 5]}
    bst = xgb.Booster(model_file=bytearray(json.dumps(doc).encode()))
    np.testing.assert_allclose(bst.predict(xgb.DMatrix(X)), [0.25, 1.0])
    lp = json.loads(bst.save_config())["learner"]["objective"]["lambdarank_param"]
    assert lp["lambdarank_pair_method"] == "mean" and lp["ndcg_exp_gain"] == "1"
    # a position-debiased model serves its margins; only training with lambdarank_unbiased=true is refused
    doc["learner"]["objective"]["lambdarank_param"]["lambdarank_unbiased"] = "1"
    biased = xgb.Booster(model_file=bytearray(json.dumps(doc).encode()))
    np.testing.assert_allclose(biased.predict(xgb.DMatrix(X)), [0.25, 1.0])
    d = xgb.DMatrix(X, label=[0, 1], group=[2])
    with pytest.raises(xgb.XGBoostError, match="lambdarank_unbiased"):
        xgb.train({}, d, 1, xgb_model=biased)


def test_combinations(xgb):
    rng = np.random.default_rng(16)
    X, y, sizes = _rank_data(rng)
    d = xgb.DMatrix(X, label=y, group=sizes)
    for extra in ({"subsample": 0.6}, {"subsample": 0.6, "sampling_method": "gradient_based"}, {"booster": "dart", "rate_drop": 0.2},
                  {"num_parallel_tree": 3, "subsample": 0.8}):
        res = {}
        bst = xgb.train(dict(objective="rank:ndcg", max_depth=3, seed=1, **extra), d, 8, evals=[(d, "t")], evals_result=res, verbose_eval=False)
        assert np.all(np.isfinite(bst.predict(d)))
        assert res["t"]["ndcg@32"][-1] > res["t"]["ndcg@32"][0], extra
    # subsample zeroes the unsampled rows of the topk gradients with the shared draw
    bst = xgb.Booster({"objective": "rank:ndcg", "subsample": 0.5, "seed": 3}, [d])
    m = rng.standard_normal(d.num_row()).astype(np.float32)
    plain = xgb.Booster({"objective": "rank:ndcg"}, [d])
    full = _be().booster_compute_gradient(plain.handle, d.handle, m)
    sub = _be().booster_compute_gradient(bst.handle, d.handle, m)
    kept = np.any(sub != 0, axis=(1, 2))
    np.testing.assert_array_equal(sub[kept], full[kept])
    assert 0.4 < kept.mean() < 0.6


def test_xgbranker(xgb):
    rng = np.random.default_rng(17)
    X, y, sizes = _rank_data(rng)
    qid = np.repeat(np.arange(len(sizes)), sizes)
    Xe, ye, se = _rank_data(rng, G=50)
    r = xgb.XGBRanker(n_estimators=10, max_depth=3)
    r.fit(X, y, qid=qid, eval_set=[(Xe, ye)], eval_group=[se])
    assert r.get_booster().save_config().find('"rank:ndcg"') > 0
    p = r.predict(X)
    np.testing.assert_array_equal(p, r.get_booster().predict(xgb.DMatrix(X), output_margin=True))
    assert len(r.evals_result()["validation_0"]["ndcg@32"]) == 10
    r2 = xgb.XGBRanker(n_estimators=10, max_depth=3).fit(X, y, group=sizes)
    np.testing.assert_array_equal(r2.predict(X), p)


def test_errors(xgb):
    rng = np.random.default_rng(18)
    X = rng.standard_normal((20, 2)).astype(np.float32)
    y = rng.integers(0, 3, 20).astype(np.float32)
    d = xgb.DMatrix(X, label=y, group=[10, 10])

    def train(params, dm=d):
        return xgb.train(params, dm, 1)
    with pytest.raises(xgb.XGBoostError, match="lambdarank_unbiased"):
        train({"objective": "rank:ndcg", "lambdarank_unbiased": True})
    with pytest.raises(xgb.XGBoostError, match="lambdarank_num_pair_per_sample"):
        train({"objective": "rank:ndcg", "lambdarank_pair_method": "mean", "lambdarank_num_pair_per_sample": 1 << 21})
    with pytest.raises(xgb.XGBoostError, match="lambdarank_pair_method"):
        train({"objective": "rank:ndcg", "lambdarank_pair_method": "all"})
    with pytest.raises(xgb.XGBoostError, match="lambdarank_num_pair_per_sample"):
        train({"objective": "rank:ndcg", "lambdarank_num_pair_per_sample": 0})
    with pytest.raises(xgb.XGBoostError, match="ndcg_exp_gain"):
        train({"objective": "rank:ndcg", "ndcg_exp_gain": "maybe"})
    with pytest.raises(xgb.XGBoostError, match="label must be 0 or 1"):
        train({"objective": "rank:map"})
    with pytest.raises(xgb.XGBoostError, match="label must be <= 31"):
        train({"objective": "rank:ndcg"}, xgb.DMatrix(X, label=np.full(20, 40.0), group=[20]))
    train({"objective": "rank:ndcg", "ndcg_exp_gain": False}, xgb.DMatrix(X, label=np.full(20, 40.0), group=[20]))
    with pytest.raises(xgb.XGBoostError, match="label must be >= 0"):
        train({"objective": "rank:ndcg"}, xgb.DMatrix(X, label=-np.ones(20), group=[20]))
    with pytest.raises(xgb.XGBoostError, match="must not be NaN"):
        train({"objective": "rank:pairwise"}, xgb.DMatrix(X, label=np.full(20, np.nan), group=[20]))
    with pytest.raises(xgb.XGBoostError, match="one weight per query group"):
        train({"objective": "rank:ndcg"}, xgb.DMatrix(X, label=y, weight=np.ones(20), group=[10, 10]))
    with pytest.raises(xgb.XGBoostError, match="ranking AUC"):
        xgb.train({"objective": "rank:ndcg", "eval_metric": "auc"}, d, 1, evals=[(d, "t")], verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="pre@k"):
        xgb.train({"objective": "rank:ndcg", "eval_metric": "pre@5"}, d, 1, evals=[(d, "t")], verbose_eval=False)
    with pytest.raises(ValueError, match="group / qid"):
        from sagemaker_xgboost_container_b200 import dask as xdask
        xdask.DaskDMatrix(None, X, y, group=[10, 10])
    # every other objective keeps reading one weight per row
    with pytest.raises(xgb.XGBoostError, match="one entry per row"):
        train({"objective": "reg:squarederror"}, xgb.DMatrix(X, label=y, weight=np.ones(2), group=[10, 10]))
    res = {}
    dl = xgb.DMatrix(X, label=(y > 0).astype(np.float32), group=[10, 10])
    xgb.train({"objective": "binary:logistic", "eval_metric": "auc"}, dl, 1, evals=[(dl, "t")], evals_result=res, verbose_eval=False)
    assert "auc" in res["t"]


TWO_RANK_PARAMS = dict(objective="rank:ndcg", max_depth=5, eta=0.3, eval_metric=["ndcg@5", "map"])


def two_rank_data():
    """Quantised features (at most 2048 distinct values per feature and shard, so the shards' cuts are the 1-GPU cuts)."""
    rng = np.random.default_rng(31)
    sizes = rng.integers(1, 60, 1200)
    n = int(sizes.sum())
    X, _ = synth(n, 10, 31, "reg")
    y = np.clip(np.round(X[:, 0] + 0.5 * X[:, 1] + 1.5 + 0.3 * rng.standard_normal(n)), 0, 4).astype(np.float32)
    w = rng.uniform(0.5, 2.0, len(sizes)).astype(np.float32)
    return X, y, sizes, w


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks(xgb, tmp_path):
    """Whole groups per rank: the 2-rank model is the 1-GPU model bit for bit (group count and weight sum all-reduced), and the
    all-reduced ndcg@5 / map equal the 1-GPU values."""
    import subprocess
    import sys
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29623", os.path.join(root, "tests", "helpers", "ranking_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y, sizes, w = two_rank_data()
    d = xgb.DMatrix(X, label=y, weight=w, group=sizes)
    single = xgb.train(TWO_RANK_PARAMS, d, num_boost_round=3, verbose_eval=False)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(xgb.Booster(model_file=out).handle)
    from util import assert_same_structure
    assert_same_structure(m2, m1)
    np.testing.assert_array_equal(m2["split_cond"].view(np.uint32), m1["split_cond"].view(np.uint32))
    one = dict(kv.split(":") for kv in single.eval_set([(d, "train")], 3).split("\t")[1:])
    with open(out + ".eval") as f:
        two = dict(kv.split(":") for kv in f.read().split("\t")[1:])
    for k in ("train-ndcg@5", "train-map"):
        assert float(two[k]) == pytest.approx(float(one[k]), rel=1e-12)
