"""reg:quantileerror on the GPU (run with `pytest -m gpu` on an H100): gradients and whole models against
tests/quantile_reference.py bit for bit, the independence of the targets, the quantile metric, prediction shapes and model IO,
forests and dart with several outputs, the error cases, the sklearn wrapper and two ranks."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import quantile_reference as QR
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
ALPHA3 = "(0.1,0.5,0.9)"


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_bits(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return a.shape == b.shape and bool(np.all((_u32(a) == _u32(b)) | (np.isnan(a) & np.isnan(b))))


def _data(n, F, seed, missing_frac=0.0):
    X, y = synth(n, F, seed, "reg", missing_frac=missing_frac)
    y = (y + np.random.default_rng(seed).laplace(0, 0.5, n)).astype(f32)
    return X, y


BASE = dict(objective="reg:quantileerror", quantile_alpha=ALPHA3, tree_method="hist", max_bin=256, max_depth=6, eta=0.3)


# ---------------------------------------------------------------------------------------------------------------- gradients
@pytest.mark.parametrize("alpha", ["0.3", ALPHA3])
@pytest.mark.parametrize("weighted", [False, True])
def test_gradient_bit_exact(xgb, alpha, weighted):
    X, y = _data(20011, 6, 1, missing_frac=0.1)
    rng = np.random.default_rng(2)
    w = rng.uniform(0, 3, len(y)).astype(f32) if weighted else None
    Q = len(QR.parse_alpha(alpha))
    m = rng.standard_normal((len(y), Q)).astype(f32)
    m[:50] = y[:50, None]                                       # d == 0
    d = xgb.DMatrix(X, label=y, weight=w)
    for extra in ({}, dict(subsample=0.5, seed=3)):
        bst = xgb.Booster(dict(BASE, quantile_alpha=alpha, **extra), [d])
        got = _be().booster_compute_gradient(bst.handle, d.handle, m, round=2)
        keep = None
        if extra:
            from forest_reference import row_mask
            keep = row_mask(3, 2, 0, len(y), 0.5)
        assert _same_bits(got, QR.gradient(m, y, QR.parse_alpha(alpha), w, keep)), extra


# ---------------------------------------------------------------------------------------------------------------- whole models
MODEL_CASES = {
    "q3": (20000, 8, {}, {}),
    "q1": (20000, 8, dict(quantile_alpha="0.25"), {}),
    "q1_weights": (20000, 8, dict(quantile_alpha="[0.8]"), dict(weighted=True)),
    "q3_weights": (20000, 8, {}, dict(weighted=True)),
    "q3_missing_depth8": (20000, 8, dict(max_depth=8), dict(missing_frac=0.15)),
    "q2_lossguide": (20000, 8, dict(quantile_alpha="(0.05,0.95)", grow_policy="lossguide", max_depth=0, max_leaves=31), {}),
    "q4_ends": (20000, 8, dict(quantile_alpha="(0,0.2,0.7,1)"), {}),
    "q3_subsample": (3000, 8, dict(subsample=0.6, min_child_weight=0, seed=3), {}),
    "q3_base_margin": (20000, 8, {}, dict(base_margin=True)),
}


@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_model_matches_reference(xgb, case):
    n, F, extra, opts = MODEL_CASES[case]
    X, y = _data(n, F, 21, opts.get("missing_frac", 0.0))
    params = dict(BASE, **extra)
    Q = len(QR.parse_alpha(params["quantile_alpha"]))
    rng = np.random.default_rng(22)
    w = rng.integers(1, 5, n).astype(f32) if opts.get("weighted") else None
    bm = rng.normal(0, 1, (n, Q)).astype(f32) if opts.get("base_margin") else None
    d = xgb.DMatrix(X, label=y, weight=w, base_margin=None if bm is None else bm.reshape(-1))
    bst = xgb.Booster(params, [d])
    ref = QR.QuantileTrainer(params, X, y, weight=w, base_margin=bm, bins=_be().dmatrix_get_bins(d.handle, 256),
                             cuts=_be().dmatrix_get_cuts(d.handle, 256))
    for r in range(4):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert m["num_class"] == Q
    assert m["base_score"] == mr["base_score"]
    assert_same_structure(m, mr)
    empty = 0
    for tid, vals in ref.leaves.items():
        off = int(mr["tree_offset"][tid])
        leaves = np.nonzero(mr["left"][off:int(mr["tree_offset"][tid + 1])] == -1)[0]
        empty += len(leaves) - len(vals)
        for nid, v in vals.items():
            assert _u32(m["split_cond"][off + nid]) == _u32(v), (tid, nid)
    assert max_leaf_diff(m, mr) <= 1e-5
    cache = _be().booster_cached_margin(bst.handle, d.handle, Q)
    if empty == 0:
        assert _same_bits(cache, ref.m)
    else:          # unsampled rows in a leaf without sampled rows take its Newton value: equal to 1e-5 per tree
        assert "subsample" in extra
        np.testing.assert_allclose(cache, ref.m, rtol=0, atol=1e-5 * 4)
    pred = bst.predict(d, output_margin=True)
    assert _same_bits(pred.reshape(n, Q), cache)


def test_base_score(xgb):
    X, y = _data(30001, 4, 31)
    for w in (None, np.random.default_rng(32).uniform(0, 4, len(y)).astype(f32)):
        bst = xgb.train(dict(BASE), xgb.DMatrix(X, label=y, weight=w), num_boost_round=1, verbose_eval=False)
        assert f32(_be().booster_export_model(bst.handle)["base_score"]) == QR.base_score(y, QR.parse_alpha(ALPHA3), w)


def test_targets_are_independent(xgb):
    """With base_score given, the trees of target j of a 3-output model are those of a 1-output model at alpha_j alone."""
    X, y = _data(20000, 8, 41)
    d = xgb.DMatrix(X, label=y)
    p = dict(BASE, base_score=0.25)
    b3 = xgb.train(p, d, num_boost_round=4, verbose_eval=False)
    m3 = _be().booster_export_model(b3.handle)
    for j, a in enumerate(QR.parse_alpha(ALPHA3)):
        b1 = xgb.train(dict(p, quantile_alpha=str(float(a))), d, num_boost_round=4, verbose_eval=False)
        m1 = _be().booster_export_model(b1.handle)
        for r in range(4):
            t3, t1 = 3 * r + j, r
            s3, e3 = int(m3["tree_offset"][t3]), int(m3["tree_offset"][t3 + 1])
            s1, e1 = int(m1["tree_offset"][t1]), int(m1["tree_offset"][t1 + 1])
            assert m3["tree_info"][t3] == j and m1["tree_info"][t1] == 0
            for k in ("left", "right", "split_index", "default_left"):
                np.testing.assert_array_equal(m3[k][s3:e3], m1[k][s1:e1], err_msg="%s target %d round %d" % (k, j, r))
            assert _same_bits(m3["split_cond"][s3:e3], m1["split_cond"][s1:e1]), (j, r)


def test_nan_label_and_bad_alpha_rejected(xgb):
    X, y = _data(200, 3, 33)
    d = xgb.DMatrix(X, label=y)
    for bad, match in ((None, "quantile_alpha"), ("[]", "quantile_alpha"), ("()", "quantile_alpha"), ("1.5", "quantile_alpha"),
                       ("(0.1,-0.2)", "quantile_alpha"), ("0.1;0.2", "quantile_alpha")):
        p = dict(BASE)
        if bad is None:
            p.pop("quantile_alpha")
        else:
            p["quantile_alpha"] = bad
        with pytest.raises(xgb.core.XGBoostError, match=match):
            xgb.train(p, d, num_boost_round=1, verbose_eval=False)
    y2 = y.copy()
    y2[7] = np.nan
    with pytest.raises(xgb.core.XGBoostError, match="must not be NaN"):
        xgb.train(dict(BASE), xgb.DMatrix(X, label=y2), num_boost_round=1, verbose_eval=False)
    with pytest.raises(xgb.core.XGBoostError):                      # two label columns
        xgb.train(dict(BASE), xgb.DMatrix(X, label=np.stack([y, y], axis=1)), num_boost_round=1, verbose_eval=False)
    # other objectives accept quantile_alpha and ignore it
    a = xgb.train(dict(objective="reg:squarederror", max_depth=3), d, num_boost_round=2, verbose_eval=False)
    b = xgb.train(dict(objective="reg:squarederror", max_depth=3, quantile_alpha="7"), d, num_boost_round=2, verbose_eval=False)
    assert _same_bits(a.predict(d), b.predict(d))
    # the quantile metric needs as many quantile_alpha values as the model has outputs
    with pytest.raises(xgb.core.XGBoostError, match="quantile"):
        xgb.train(dict(objective="reg:squarederror", quantile_alpha="(0.1,0.9)", eval_metric="quantile"), d, num_boost_round=1,
                  evals=[(d, "train")], verbose_eval=False)


# ---------------------------------------------------------------------------------------------------------------- metric
@pytest.mark.parametrize("weighted", [False, True])
def test_quantile_metric(xgb, weighted):
    X, y = _data(20000, 6, 51)
    w = np.random.default_rng(52).uniform(0, 2, len(y)).astype(f32) if weighted else None
    d = xgb.DMatrix(X, label=y, weight=w)
    res = {}
    bst = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=3, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    assert list(res["train"]) == ["quantile"]
    pred = bst.predict(d)
    assert abs(res["train"]["quantile"][-1] - QR.pinball(y, pred, QR.parse_alpha(ALPHA3), w)) <= 2e-5
    # a squared-error model evaluated with the metric at one alpha
    sq = xgb.train(dict(objective="reg:squarederror", max_depth=4, quantile_alpha="0.7", eval_metric="quantile"), d, num_boost_round=2,
                   evals=[(d, "train")], evals_result=res, verbose_eval=False)
    assert abs(res["train"]["quantile"][-1] - QR.pinball(y, sq.predict(d), [0.7], w)) <= 2e-5


# ---------------------------------------------------------------------------------------------------------------- prediction
def test_prediction_shapes_and_ranges(xgb):
    X, y = _data(3000, 5, 61)
    d = xgb.DMatrix(X, label=y)
    b1 = xgb.train(dict(BASE, quantile_alpha="0.5", max_depth=4), d, num_boost_round=4, verbose_eval=False)
    assert b1.predict(d).shape == (3000,) and b1.predict(d, strict_shape=True).shape == (3000, 1)
    b3 = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=4, verbose_eval=False)
    p3 = b3.predict(d)
    assert p3.shape == (3000, 3) and b3.predict(d, strict_shape=True).shape == (3000, 3)
    assert _same_bits(p3, b3.predict(d, output_margin=True))                  # the identity transform
    # quantiles in order on average (the targets are fitted independently)
    assert np.mean(p3[:, 0]) < np.mean(p3[:, 1]) < np.mean(p3[:, 2])
    leaf = b3.predict(d, pred_leaf=True)
    assert leaf.shape == (3000, 12)
    part = b3.predict(d, iteration_range=(1, 3))
    assert _same_bits(b3[1:3].predict(d), part)
    assert b3[1:3].predict(d, pred_leaf=True).shape == (3000, 6)
    np.testing.assert_array_equal(b3[1:3].predict(d, pred_leaf=True), leaf[:, 3:9])
    contrib = b3.predict(d, pred_contribs=True)
    assert contrib.shape == (3000, 3, 6)
    np.testing.assert_allclose(contrib.sum(axis=2), p3, rtol=0, atol=1e-5)


def test_model_io_round_trips(xgb, tmp_path):
    X, y = _data(5000, 6, 62)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=4, verbose_eval=False)
    p0 = bst.predict(d)
    for fmt in ("json", "ubj"):
        path = str(tmp_path / ("m." + fmt))
        bst.save_model(path)
        assert _same_bits(xgb.Booster(model_file=path).predict(d), p0)
    assert _same_bits(pickle.loads(pickle.dumps(bst)).predict(d), p0)
    doc = json.loads(open(str(tmp_path / "m.json")).read())
    assert doc["learner"]["objective"] == {"name": "reg:quantileerror", "quantile_loss_param": {"quantile_alpha": "[0.1, 0.5, 0.9]"}}
    assert doc["learner"]["learner_model_param"]["num_target"] == "3" and doc["learner"]["learner_model_param"]["num_class"] == "0"
    assert doc["learner"]["gradient_booster"]["model"]["tree_info"] == [0, 1, 2] * 4
    cfg = bst.save_config()
    assert json.loads(cfg)["learner"]["learner_model_param"]["num_target"] == "3"
    fresh = xgb.Booster()
    fresh.load_model(str(tmp_path / "m.ubj"))
    fresh.load_config(cfg)
    assert _same_bits(fresh.predict(d), p0)
    # training continues from a loaded document as from the booster it was saved from
    cont = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=2, xgb_model=str(tmp_path / "m.json"), verbose_eval=False)
    full = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=6, verbose_eval=False)
    assert _same_bits(cont.predict(d), full.predict(d))
    # a document whose num_target disagrees with quantile_alpha is refused
    doc["learner"]["learner_model_param"]["num_target"] = "2"
    bad = str(tmp_path / "bad.json")
    with open(bad, "w") as f:
        json.dump(doc, f)
    with pytest.raises(xgb.core.XGBoostError, match="num_target"):
        xgb.Booster(model_file=bad)


@pytest.mark.parametrize("extra", [dict(num_parallel_tree=2, subsample=0.7, colsample_bynode=0.8, seed=5),
                                   dict(num_parallel_tree=2, seed=6),
                                   dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7)])
def test_forest_and_dart_cache_equals_predict(xgb, extra):
    X, y = _data(20000, 8, 71)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(dict(BASE, quantile_alpha="(0.2,0.8)", **extra), [d])
    for r in range(4):
        bst.update(d, r)
    P = int(extra.get("num_parallel_tree", 1))
    m = _be().booster_export_model(bst.handle)
    np.testing.assert_array_equal(m["tree_info"], np.repeat(np.tile(np.arange(2), 1), P).tolist() * 4)
    cache = _be().booster_cached_margin(bst.handle, d.handle, 2)
    pred = bst.predict(d, output_margin=True)
    if extra.get("booster") == "dart":        # predict sums fl(w_t * leaf_t) afresh; the cache carries each round's weight changes
        np.testing.assert_allclose(pred, cache, rtol=0, atol=1e-5)
    else:
        assert _same_bits(pred, cache)
    assert bst.predict(d, pred_leaf=True).shape == (20000, 4 * 2 * P)


def test_sklearn_regressor(xgb):
    X, y = _data(5000, 6, 81)
    from sagemaker_xgboost_container_b200 import sklearn as skl
    for alpha in ([0.1, 0.9], np.array([0.1, 0.9]), (0.1, 0.9)):
        reg = skl.XGBRegressor(objective="reg:quantileerror", quantile_alpha=alpha, n_estimators=3, max_depth=4)
        reg.fit(X, y)
        p = reg.predict(X)
        assert p.shape == (5000, 2)
    params = {"objective": "reg:quantileerror", "quantile_alpha": "[0.1, 0.9]", "max_depth": "4", "eta": "0.3"}
    bst = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    assert _same_bits(bst.predict(xgb.DMatrix(X)), p)


# ---------------------------------------------------------------------------------------------------------------- two ranks
def test_two_ranks(xgb, tmp_path):
    """Two ranks train the 1-GPU model bit for bit: the labels' quantiles and the leaves' are exact over both ranks' rows."""
    try:
        import torch
        ngpu = torch.cuda.device_count()
    except Exception:
        ngpu = 0
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    n, F, rounds = 40000, 20, 4
    extra = dict(quantile_alpha=ALPHA3, seed=3)
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29621", os.path.join(ROOT, "tests", "helpers", "train_shard_worker.py"), out, str(n), str(F), str(rounds), "reg:quantileerror", repr(extra)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y = synth(n, F, 7, "reg")
    single = xgb.train(dict(dict(objective="reg:quantileerror", max_depth=5, eta=0.3, max_bin=256), **extra), xgb.DMatrix(X, label=y),
                       num_boost_round=rounds, verbose_eval=False)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(xgb.Booster(model_file=out).handle)
    assert m1["base_score"] == m2["base_score"]
    assert_same_structure(m2, m1)
    assert _same_bits(m2["split_cond"], m1["split_cond"])
