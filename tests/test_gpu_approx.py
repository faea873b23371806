"""tree_method=approx on the GPU: the cuts every tree grows on against the shared cut rule with that tree's hessian
(tests/cuts_reference.py), whole models against tests/approx_reference.py, hist trees for constant-hessian objectives,
determinism, resumed training, the matrix's own bins after approx, custom objectives and the QuantileDMatrix refusal."""
import json

import numpy as np
import pytest

import approx_reference as AR
import cuts_reference as CR
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ARRAYS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")
MAX_BIN = 64


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_model(a, b):
    for k in ARRAYS:
        x, y = (a[k], b[k]) if a[k].dtype != np.float32 else (_u32(a[k]), _u32(b[k]))
        np.testing.assert_array_equal(x, y, err_msg=k)


def _data(kind="bin", K=1, n=4000, F=8, seed=11, missing=0.04):
    X, y = synth(n, F, seed, kind, K=K, quantised=False, missing_frac=missing)
    X[:, F - 1] = np.round(X[:, F - 1] * 2) + np.float32(0)     # fewer distinct values than bins: its cuts never move
    return X, y


def _weights(n, seed=5):
    return np.random.default_rng(seed).uniform(0.5, 2.0, n).astype(np.float32)


def _train(xgb, d, params, rounds, record=True):
    bst = xgb.Booster(params, [d])
    if record:
        _be().booster_set_record_cuts(bst.handle, True)
    margins = []
    for r in range(rounds):
        margins.append(_be().booster_training_margin(bst.handle, d.handle))
        bst.update(d, r)
    return bst, margins


def _check_tree_cuts(xgb, X, d, bst, margins, params, P=1):
    """each tree's cuts are the cut rule with its class's hessian at the round's starting margin, before row sampling"""
    plain = xgb.Booster({k: v for k, v in params.items() if k not in ("subsample", "sampling_method")}, [d])
    t = 0
    for r, m in enumerate(margins):
        gp = _be().booster_compute_gradient(plain.handle, d.handle, m, r)
        for k in range(gp.shape[1]):
            ref = CR.make_cuts(X, MAX_BIN, gp[:, k, 1])
            for _ in range(P):
                got = _be().booster_tree_cuts(bst.handle, t)
                np.testing.assert_array_equal(got[0], ref[0], err_msg="tree %d" % t)
                np.testing.assert_array_equal(_u32(got[1]), _u32(ref[1]), err_msg="tree %d" % t)
                np.testing.assert_array_equal(_u32(got[2]), _u32(ref[2]), err_msg="tree %d" % t)
                t += 1
    assert t == len(_be().booster_export_model(bst.handle)["tree_info"])


def _base(objective, **kw):
    p = dict(objective=objective, tree_method="approx", max_bin=MAX_BIN, max_depth=5, eta=0.5, base_score=0.5, seed=3)
    p.update(kw)
    return p


# ---- constant hessian: approx grows hist trees
@pytest.mark.parametrize("case", ["squarederror", "squarederror-weights", "absoluteerror", "quantileerror"])
def test_constant_hessian_equals_hist(xgb, case):
    X, y = _data("reg")
    w = _weights(len(y)) if case.endswith("weights") else None
    obj = {"squarederror": "reg:squarederror", "squarederror-weights": "reg:squarederror", "absoluteerror": "reg:absoluteerror",
           "quantileerror": "reg:quantileerror"}[case]
    extra = dict(quantile_alpha=0.3) if case == "quantileerror" else {}
    models = []
    for tm in ("hist", "approx"):
        d = xgb.DMatrix(X, label=y, weight=w)
        bst = xgb.train(dict(_base(obj, **extra), tree_method=tm), d, num_boost_round=4)
        models.append(_be().booster_export_model(bst.handle))
    _same_model(models[0], models[1])


# ---- per-tree cuts
def _objective_case(xgb, case):
    n = 4000
    if case == "logistic":
        X, y = _data("bin")
        return X, xgb.DMatrix(X, label=y, weight=_weights(n)), _base("binary:logistic")
    if case == "softprob":
        X, y = _data("multi", K=3)
        return X, xgb.DMatrix(X, label=y, weight=_weights(n)), _base("multi:softprob", num_class=3)
    if case == "poisson":
        X, y = _data("count")
        return X, xgb.DMatrix(X, label=y, weight=_weights(n)), _base("count:poisson")
    if case == "pseudohuber":
        X, y = _data("reg")
        return X, xgb.DMatrix(X, label=y, weight=_weights(n)), _base("reg:pseudohubererror")
    if case == "aft":
        X, y = _data("pos")
        lo = y.astype(np.float32)
        hi = np.where(np.arange(n) % 4 == 0, np.float32(np.inf), lo * 1.5).astype(np.float32)
        return X, xgb.DMatrix(X, weight=_weights(n), label_lower_bound=lo, label_upper_bound=hi), _base("survival:aft")
    if case == "ndcg":
        X, y = _data("count")
        y = np.minimum(y, 4).astype(np.float32)
        d = xgb.DMatrix(X, label=y)
        sizes = [40] * (n // 40)
        d.set_group(sizes)
        d.set_weight(_weights(len(sizes)))
        return X, d, _base("rank:ndcg", ndcg_exp_gain=False)
    raise ValueError(case)


@pytest.mark.parametrize("case", ["logistic", "softprob", "poisson", "pseudohuber", "aft", "ndcg"])
def test_tree_cuts_are_the_hessian_cuts(xgb, case):
    X, d, params = _objective_case(xgb, case)
    bst, margins = _train(xgb, d, params, 3)
    _check_tree_cuts(xgb, X, d, bst, margins, params)


# ---- whole models against the restatement
SWEEP = {
    "logistic": ("binary:logistic", "bin", 1, 1, {}),
    "softprob": ("multi:softprob", "multi", 3, 1, {}),
    "subsample": ("binary:logistic", "bin", 1, 1, dict(subsample=0.7)),
    "forest": ("binary:logistic", "bin", 1, 3, dict(subsample=0.8)),
    "lossguide": ("binary:logistic", "bin", 1, 1, dict(grow_policy="lossguide", max_leaves=12, max_depth=0)),
    "monotone": ("binary:logistic", "bin", 1, 1, dict(monotone_constraints="(1,-1,0,0,1,0,0,0)")),
    "colsample": ("binary:logistic", "bin", 1, 1, dict(colsample_bytree=0.7, colsample_bynode=0.8)),
    "interaction": ("binary:logistic", "bin", 1, 1, dict(interaction_constraints="[[0, 1, 2], [3, 4, 5, 6, 7]]")),
}


@pytest.mark.parametrize("case", sorted(SWEEP))
def test_models_match_the_restatement(xgb, oracle, case):
    objective, kind, K, P, extra = SWEEP[case]
    X, y = _data(kind, K=K, n=3000, missing=0.02)
    w = _weights(len(y))
    params = _base(objective, num_parallel_tree=P, **extra)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y, weight=w)
    bst, margins = _train(xgb, d, params, 3)
    ref = AR.ApproxTrainer(params, X, y, P=P, weights=w, base_score=0.5)
    for _ in range(3):
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= 1e-5
    for t, c in enumerate(ref.tree_cuts):
        got = _be().booster_tree_cuts(bst.handle, t)
        np.testing.assert_array_equal(got[0], c[0], err_msg="tree %d" % t)
        np.testing.assert_array_equal(_u32(got[1]), _u32(c[1]), err_msg="tree %d" % t)
    _check_tree_cuts(xgb, X, d, bst, margins, params, P)


def test_gradient_based_sampling_sketches_unsampled_hessians(xgb):
    X, y = _data("bin")
    params = _base("binary:logistic", subsample=0.5, sampling_method="gradient_based")
    d = xgb.DMatrix(X, label=y, weight=_weights(len(y)))
    bst, margins = _train(xgb, d, params, 3)
    _check_tree_cuts(xgb, X, d, bst, margins, params)


def test_zero_total_weight(xgb):
    """Every hessian 0 (as a saturated logistic gives): each wide feature's cuts are its second value and the end cut."""
    X, y = _data("bin", missing=0.0)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(_base("binary:logistic", max_depth=2), [d])
    _be().booster_set_record_cuts(bst.handle, True)
    h = np.zeros(len(y), np.float32)
    bst.boost(d, 0, np.full(len(y), 0.5, np.float32), h)
    got = _be().booster_tree_cuts(bst.handle, 0)
    ref = CR.make_cuts(X, MAX_BIN, h)
    np.testing.assert_array_equal(got[0], ref[0])
    np.testing.assert_array_equal(_u32(got[1]), _u32(ref[1]))
    for f in range(X.shape[1] - 1):
        dv = np.unique(X[:, f])
        np.testing.assert_array_equal(_u32(got[1][got[0][f]:got[0][f + 1]]), _u32([dv[1], CR.end_cut(dv[-1])]))


# ---- determinism and reuse
def test_two_runs_same_bytes(xgb):
    X, y = _data("multi", K=3)
    params = _base("multi:softprob", num_class=3, subsample=0.8)
    raws = [xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=4).save_raw("ubj") for _ in range(2)]
    assert raws[0] == raws[1]


def test_resume_equals_one_go(xgb):
    X, y = _data("bin")
    params = _base("binary:logistic")
    d = xgb.DMatrix(X, label=y)
    whole = xgb.train(params, d, num_boost_round=6)
    first = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=3)
    loaded = xgb.Booster(params)
    loaded.load_model(bytearray(first.save_raw("ubj")))
    resumed = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=3, xgb_model=loaded)
    assert resumed.save_raw("ubj") == whole.save_raw("ubj")


def test_config_round_trips(xgb):
    X, y = _data("bin")
    bst = xgb.train(_base("binary:logistic"), xgb.DMatrix(X, label=y), num_boost_round=1)
    cfg = json.loads(bst.save_config())
    gtp = cfg["learner"]["gradient_booster"]["gbtree_train_param"]
    assert gtp["tree_method"] == "approx"
    other = xgb.Booster()
    other.load_config(bst.save_config())
    assert json.loads(other.save_config())["learner"]["gradient_booster"]["gbtree_train_param"]["tree_method"] == "approx"


def test_hist_after_approx_uses_the_matrix_own_bins(xgb):
    X, y = _data("bin")
    hist = dict(_base("binary:logistic"), tree_method="hist")
    d = xgb.DMatrix(X, label=y)
    xgb.train(_base("binary:logistic"), d, num_boost_round=2)
    after = xgb.train(hist, d, num_boost_round=3)
    fresh = xgb.train(hist, xgb.DMatrix(X, label=y), num_boost_round=3)
    assert after.save_raw("ubj") == fresh.save_raw("ubj")
    # a QuantileDMatrix built with it as ref takes its own cuts, not the last tree's
    dq = xgb.QuantileDMatrix(X, ref=d, max_bin=MAX_BIN)
    ref_cuts = _be().dmatrix_get_cuts(d.handle, MAX_BIN)
    own = CR.make_cuts(X, MAX_BIN)
    np.testing.assert_array_equal(_u32(ref_cuts[1]), _u32(own[1]))
    np.testing.assert_array_equal(fresh.predict(dq), after.predict(dq))


def test_custom_objective_resketches_from_the_callers_hessian(xgb):
    X, y = _data("reg")
    params = _base("reg:squarederror")
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    _be().booster_set_record_cuts(bst.handle, True)
    rng = np.random.default_rng(9)
    hs = []
    for r in range(2):
        m = bst.predict(d, output_margin=True)
        g = (m - y).astype(np.float32)
        h = rng.uniform(0.25, 1.0, len(y)).astype(np.float32)
        hs.append(h)
        bst.boost(d, r, g, h)
    for t, h in enumerate(hs):
        got = _be().booster_tree_cuts(bst.handle, t)
        ref = CR.make_cuts(X, MAX_BIN, h)
        np.testing.assert_array_equal(got[0], ref[0])
        np.testing.assert_array_equal(_u32(got[1]), _u32(ref[1]))


def test_quantile_dmatrix_refused_and_exact_warns(xgb):
    X, y = _data("bin")
    dq = xgb.QuantileDMatrix(X, label=y, max_bin=MAX_BIN)
    with pytest.raises(xgb.core.XGBoostError, match="tree_method=approx"):
        xgb.train(_base("binary:logistic"), dq, num_boost_round=1)
    with pytest.warns(UserWarning, match="tree_method=exact"):
        xgb.train(dict(_base("binary:logistic"), tree_method="exact"), xgb.DMatrix(X, label=y), num_boost_round=1)


def test_dart_resketches_each_tree(xgb):
    """booster=dart: the first round drops nothing, so its tree's cuts are the cut rule at the base margin; later rounds take
    the hessian at the margin without the dropped trees, and the run is deterministic."""
    X, y = _data("bin")
    params = _base("binary:logistic", booster="dart", rate_drop=0.5, seed=4)
    d = xgb.DMatrix(X, label=y, weight=_weights(len(y)))
    bst, margins = _train(xgb, d, params, 4)
    plain = xgb.Booster({k: v for k, v in params.items() if k not in ("booster", "rate_drop")}, [d])
    h0 = _be().booster_compute_gradient(plain.handle, d.handle, margins[0], 0)[:, 0, 1]
    ref = CR.make_cuts(X, MAX_BIN, h0)
    got = _be().booster_tree_cuts(bst.handle, 0)
    np.testing.assert_array_equal(got[0], ref[0])
    np.testing.assert_array_equal(_u32(got[1]), _u32(ref[1]))
    again, _ = _train(xgb, xgb.DMatrix(X, label=y, weight=_weights(len(y))), params, 4)
    assert again.save_raw("ubj") == bst.save_raw("ubj")
    hist = xgb.train(dict(params, tree_method="hist"), xgb.DMatrix(X, label=y, weight=_weights(len(y))), num_boost_round=4)
    assert hist.save_raw("ubj") != bst.save_raw("ubj")


def test_set_cuts_survives_approx(xgb):
    """External cuts (XGB200DMatrixSetCuts): an approx booster re-sketches from the data, and a hist booster afterwards grows on
    the external cuts again, not on cuts recomputed from the data."""
    X, y = _data("bin")
    coarse = CR.make_cuts(X, 16)
    def fresh():
        d = xgb.DMatrix(X, label=y)
        _be().dmatrix_set_cuts(d.handle, coarse[0], coarse[1], coarse[2])
        return d
    hist = dict(_base("binary:logistic"), tree_method="hist")
    d = fresh()
    bst, _ = _train(xgb, d, _base("binary:logistic"), 2)
    got = _be().booster_tree_cuts(bst.handle, 0)
    assert len(got[1]) > len(coarse[1])           # the wide features took MAX_BIN hessian cuts
    after = xgb.train(hist, d, num_boost_round=2)
    assert after.save_raw("ubj") == xgb.train(hist, fresh(), num_boost_round=2).save_raw("ubj")


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_rank_approx_equals_single_gpu(xgb, tmp_path):
    """Rows sharded over 2 ranks, 256 levels per feature (at most 2048 distinct values per shard, so every rank's summary is
    exact): each tree's merged hessian cuts, and so the model, equal one GPU's, bit for bit."""
    import os
    import subprocess
    import sys
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n, F, rounds = 40000, 12, 3
    extra = dict(tree_method="approx", max_bin=MAX_BIN, base_score=0.5, seed=5)
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29617", os.path.join(root, "tests", "helpers", "train_shard_worker.py"), out, str(n), str(F), str(rounds), "binary:logistic", repr(extra)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y = synth(n, F, 7, "bin")
    single = xgb.train(dict(objective="binary:logistic", max_depth=5, eta=0.3, **extra), xgb.DMatrix(X, label=y), num_boost_round=rounds)
    multi = xgb.Booster(model_file=out)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(multi.handle)
    assert_same_structure(m2, m1)
    np.testing.assert_array_equal(_u32(m2["split_cond"]), _u32(m1["split_cond"]))
