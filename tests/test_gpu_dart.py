"""booster=dart on the GPU against the DART restatement in tests/dart_reference.py: the drop sets and tree weights bit for
bit after every round, the trees, the training cache, weighted prediction and SHAP, the dart model document."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import dart_reference as DR
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARRAYS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")
LEAF_TOL = 1e-5
MARGIN_TOL = 2e-5


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _weights(bst):
    return _be().booster_tree_weights(bst.handle)


def _pair(xgb, oracle, X, y, params, exact):
    """The product's Booster and the reference trainer on the same cuts (exact: the oracle on the device's bins and grid)."""
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    if exact:
        cuts = _be().dmatrix_get_cuts(d.handle, 256)
        bins = _be().dmatrix_get_bins(d.handle, 256)
        t = oracle.Trainer(params, bins=bins, cuts=cuts, y=y, base_score=params["base_score"])
        t.set_device_grid(X.shape[0])
        ref = DR.DartTrainer(params, X, trainer=t)
    else:
        ref = DR.DartTrainer(params, X, y)
    return d, bst, ref


def _train_and_compare(xgb, oracle, X, y, params, rounds, exact):
    d, bst, ref = _pair(xgb, oracle, X, y, params, exact)
    K = ref.K
    dropped = 0
    for r in range(rounds):
        bst.update(d, r)
        D = ref.update()
        dropped += len(D)
        np.testing.assert_array_equal(_u32(_weights(bst)), _u32(ref.weights), err_msg="round %d: weight_drop" % r)
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    cache = _be().booster_cached_margin(bst.handle, d.handle, K)
    if exact:
        for k in ARRAYS:
            np.testing.assert_array_equal(_u32(m[k]) if m[k].dtype == np.float32 else m[k], _u32(mr[k]) if mr[k].dtype == np.float32 else mr[k], err_msg=k)
        np.testing.assert_array_equal(_u32(cache), _u32(ref.m_full))
    else:
        assert max_leaf_diff(m, mr) <= LEAF_TOL
        np.testing.assert_allclose(cache, ref.m_full, rtol=0, atol=MARGIN_TOL)
    return d, bst, ref, m, dropped


def test_rate_drop_zero_is_gbtree(xgb):
    X, y = synth(20000, 28, 3, "reg")
    base = dict(objective="reg:squarederror", max_depth=6, eta=0.3, max_bin=256)
    d1, d2 = xgb.DMatrix(X, label=y), xgb.DMatrix(X, label=y)
    g = xgb.train(base, d1, num_boost_round=8, verbose_eval=False)
    b = xgb.train(dict(base, booster="dart", rate_drop=0.0, one_drop=0), d2, num_boost_round=8, verbose_eval=False)
    mg, mb = _be().booster_export_model(g.handle), _be().booster_export_model(b.handle)
    for k in ARRAYS:
        np.testing.assert_array_equal(mg[k], mb[k], err_msg=k)
    np.testing.assert_array_equal(_weights(b), np.ones(8, np.float32))
    np.testing.assert_array_equal(_u32(_be().booster_cached_margin(g.handle, d1.handle, 1)), _u32(_be().booster_cached_margin(b.handle, d2.handle, 1)))
    np.testing.assert_array_equal(_u32(g.predict(d1, output_margin=True)), _u32(b.predict(d2, output_margin=True)))
    np.testing.assert_array_equal(g.predict(d1, pred_leaf=True), b.predict(d2, pred_leaf=True))
    assert json.loads(b.save_config())["learner"]["gradient_booster"]["name"] == "dart"


DART_CASES = [dict(sample_type=s, normalize_type=nt, one_drop=od) for s in ("uniform", "weighted") for nt in ("tree", "forest") for od in (0, 1)]
DART_CASES.append(dict(sample_type="uniform", normalize_type="tree", one_drop=1, skip_drop=0.4))


@pytest.mark.parametrize("dp", DART_CASES, ids=lambda p: "-".join("%s=%s" % kv for kv in sorted(p.items())))
def test_squarederror_bit_exact_against_reference(xgb, oracle, dp):
    """reg:squarederror on quantised data with the oracle on the device's grid: weights, trees and cache equal as bits."""
    X, y = synth(12000, 20, 5, "reg")
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=5, eta=0.3, base_score=0.5, seed=7,
                  booster="dart", rate_drop=0.3, **dp)
    d, bst, ref, m, dropped = _train_and_compare(xgb, oracle, X, y, params, 20, exact=True)
    assert dropped > 0
    if dp["one_drop"] and not dp.get("skip_drop"):
        assert all(len(D) >= 1 for D in ref.drops[1:])


@pytest.mark.parametrize("objective,kind,K,extra", [
    ("binary:logistic", "bin", 1, {}),
    ("multi:softprob", "multi", 3, {}),
    ("reg:squarederror", "reg", 1, dict(grow_policy="lossguide", max_leaves=16, max_depth=0)),
    ("reg:squarederror", "reg", 1, dict(subsample=0.8, colsample_bytree=0.8, colsample_bylevel=0.7, colsample_bynode=0.7)),
])
def test_objectives_and_sampling_against_reference(xgb, oracle, objective, kind, K, extra):
    X, y = synth(10000, 16, 9, kind, K=K)
    params = dict(dict(objective=objective, tree_method="hist", max_bin=256, max_depth=4, eta=0.3, seed=5, booster="dart", rate_drop=0.3,
                       sample_type="weighted", normalize_type="forest"), **extra)
    if K > 1:
        params["num_class"] = K
    _, _, ref, m, dropped = _train_and_compare(xgb, oracle, X, y, params, 12, exact=False)
    assert dropped > 0
    assert len(m["tree_info"]) == 12 * K


def _dart_model(xgb, oracle, rounds=15, K=1, rate=0.4):
    kind = "multi" if K > 1 else "reg"
    X, y = synth(6000, 8, 13, kind, K=K)
    params = dict(objective="multi:softprob" if K > 1 else "reg:squarederror", max_depth=4, eta=0.3, max_bin=256, seed=3,
                  booster="dart", rate_drop=rate, one_drop=1)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    m["objective"] = params["objective"]
    return X, y, d, bst, m, _weights(bst)


@pytest.mark.parametrize("K", [1, 3])
def test_weighted_predict_and_contribs(xgb, oracle, K):
    X, y, d, bst, m, w = _dart_model(xgb, oracle, K=K)
    assert (w != 1).any()
    n, R = X.shape[0], 15
    for b, e in [(0, 0), (0, 5), (3, 11), (14, 15)]:
        got = bst.predict(d, output_margin=True, iteration_range=(b, e)).reshape(n, K)
        ref = DR.predict_margin(m, X, w, b * K, (e or R) * K)
        np.testing.assert_array_equal(_u32(got), _u32(ref), err_msg="iteration_range %s" % ((b, e),))
    val = bst.predict(d).reshape(n, K)
    np.testing.assert_allclose(val, oracle.transform(m, DR.predict_margin(m, X, w)).reshape(n, K), rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(bst.predict(d, training=True), bst.predict(d))
    np.testing.assert_array_equal(bst.predict(d, pred_leaf=True).astype(np.int32), oracle.predict_leaf(m, X))
    sub = X[:64]
    contrib = bst.predict(xgb.DMatrix(sub), pred_contribs=True).reshape(64, K, -1)
    np.testing.assert_allclose(contrib, DR.shap_weighted(m, sub, w), rtol=0, atol=1e-4)
    np.testing.assert_allclose(contrib.sum(axis=2), bst.predict(xgb.DMatrix(sub), output_margin=True).reshape(64, K), rtol=0, atol=1e-4)


def test_cache_and_eval_after_many_drops(xgb):
    """Incremental cache updates reorder float sums against predict(): stated bound 1e-4 on the margins after 50 rounds."""
    X, y = synth(20000, 12, 17, "reg")
    Xv, yv = synth(5000, 12, 18, "reg")
    d, dv = xgb.DMatrix(X, label=y), xgb.DMatrix(Xv, label=yv)
    res = {}
    bst = xgb.train(dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256, booster="dart", rate_drop=0.5), d,
                    num_boost_round=50, evals=[(dv, "val")], evals_result=res, verbose_eval=False)
    cache = _be().booster_cached_margin(bst.handle, d.handle, 1)[:, 0]
    pred = bst.predict(d, output_margin=True)
    assert np.abs(cache - pred).max() < 1e-4
    cv = _be().booster_cached_margin(bst.handle, dv.handle, 1)[:, 0]
    assert np.abs(cv - bst.predict(dv, output_margin=True)).max() < 1e-4
    rmse = float(np.sqrt(np.mean((bst.predict(dv).astype(np.float64) - yv) ** 2)))
    assert abs(res["val"]["rmse"][-1] - rmse) < 1e-4


def test_model_io_round_trips(xgb, oracle, tmp_path):
    X, y, d, bst, m, w = _dart_model(xgb, oracle)
    want = bst.predict(d, output_margin=True)
    for name in ("m.ubj", "m.json"):
        p = str(tmp_path / name)
        bst.save_model(p)
        b2 = xgb.Booster(model_file=p)
        np.testing.assert_array_equal(_u32(b2.predict(d, output_margin=True)), _u32(want))
        np.testing.assert_array_equal(_u32(_weights(b2)), _u32(w))
    doc = json.loads(bytes(bst.save_raw("json")))
    gb = doc["learner"]["gradient_booster"]
    assert gb["name"] == "dart" and len(gb["weight_drop"]) == len(w) and gb["gbtree"]["name"] == "gbtree"
    cfg = json.loads(bst.save_config())
    assert cfg["learner"]["learner_train_param"]["booster"] == "dart" and "dart_train_param" in cfg["learner"]["gradient_booster"]
    b3 = pickle.loads(pickle.dumps(bst))
    np.testing.assert_array_equal(_u32(b3.predict(d, output_margin=True)), _u32(want))
    sl = bst[2:9]
    np.testing.assert_array_equal(_u32(_weights(sl)), _u32(w[2:9]))
    np.testing.assert_array_equal(_u32(sl.predict(d, output_margin=True).reshape(-1, 1)), _u32(DR.predict_margin(m, X, w, 2, 9)))
    # a document written by hand with other weights predicts base + sum w * leaf
    gb["weight_drop"] = [float(v) for v in np.linspace(0.25, 2.0, len(w))]
    hw = xgb.Booster(); hw.load_model(bytearray(json.dumps(doc).encode()))
    np.testing.assert_array_equal(_u32(hw.predict(d, output_margin=True).reshape(-1, 1)), _u32(DR.predict_margin(m, X, np.float32(gb["weight_drop"]))))
    for bad in (gb["weight_drop"][:-1], gb["weight_drop"][:-1] + [float("nan")], "x"):
        doc2 = json.loads(json.dumps(doc)); doc2["learner"]["gradient_booster"]["weight_drop"] = bad
        with pytest.raises(xgb.XGBoostError):
            xgb.Booster().load_model(bytearray(json.dumps(doc2).encode()))


def test_checkpoint_resume_draws_the_same(xgb, oracle, tmp_path):
    X, y = synth(8000, 10, 21, "reg")
    params = dict(objective="reg:squarederror", max_depth=4, eta=0.3, max_bin=256, seed=9, booster="dart", rate_drop=0.3)
    d = xgb.DMatrix(X, label=y)
    full = xgb.train(params, d, num_boost_round=20, verbose_eval=False)
    first = xgb.train(params, d, num_boost_round=10, verbose_eval=False)
    p = str(tmp_path / "ckpt.ubj")
    first.save_model(p)
    resumed = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=10, xgb_model=p, verbose_eval=False)
    mf, mr = _be().booster_export_model(full.handle), _be().booster_export_model(resumed.handle)
    assert_same_structure(mr, mf)
    assert max_leaf_diff(mr, mf) <= LEAF_TOL
    wf, wr = _weights(full), _weights(resumed)
    np.testing.assert_array_equal(wf != 1, wr != 1)          # same drop sets
    np.testing.assert_allclose(wr, wf, rtol=1e-6)


@pytest.mark.parametrize("bad", [dict(sample_type="gaussian"), dict(normalize_type="none"), dict(rate_drop=1.5), dict(skip_drop=-0.1), dict(one_drop=2)])
def test_bad_parameters_raise(xgb, bad):
    X, y = synth(500, 4, 1, "reg")
    with pytest.raises(xgb.XGBoostError):
        xgb.train(dict(objective="reg:squarederror", booster="dart", **bad), xgb.DMatrix(X, label=y), num_boost_round=1, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError):
        xgb.train(dict(objective="reg:squarederror", booster="gblinear"), xgb.DMatrix(X, label=y), num_boost_round=1, verbose_eval=False)


def test_two_rank_dart_equals_single_gpu(xgb, tmp_path):
    try:
        import torch
        ngpu = torch.cuda.device_count()
    except Exception:
        ngpu = 0
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    n, F, rounds = 40000, 20, 8
    extra = dict(booster="dart", rate_drop=0.3, one_drop=1, seed=4)
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29613", os.path.join(ROOT, "tests", "helpers", "train_shard_worker.py"), out, str(n), str(F), str(rounds), "reg:squarederror", repr(extra)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y = synth(n, F, 7, "reg")
    single = xgb.train(dict(dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256), **extra), xgb.DMatrix(X, label=y),
                       num_boost_round=rounds, verbose_eval=False)
    multi = xgb.Booster(model_file=out)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(multi.handle)
    assert_same_structure(m2, m1)
    np.testing.assert_array_equal(m2["split_cond"], m1["split_cond"])
    np.testing.assert_array_equal(_u32(_weights(multi)), _u32(_weights(single)))
