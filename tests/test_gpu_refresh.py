"""process_type=update on the GPU (csrc/refresh.cu): refresh and prune of existing trees, against the NumPy restatement
(tests/refresh_reference.py) bit for bit, and the identity of refreshing a model on its own training data."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import refresh_reference as R
from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = ("sum_hess", "base_weight", "loss_chg", "split_cond")


def _export(xgb, bst):
    return xgb.get_backend().booster_export_model(bst.handle)


def _assert_models_equal(a, b, fields=R.FIELDS + ("tree_offset", "tree_info")):
    for k in fields:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def _update_params(params, updater="refresh", **kw):
    return dict(params, process_type="update", updater=updater, **kw)


IDENTITY = {
    "sqerr-dense-g": ("reg", 1, dict(objective="reg:squarederror", max_depth=6), {}),
    "logistic-weights-missing": ("bin", 1, dict(objective="binary:logistic", max_depth=5), dict(weights=True, missing_frac=0.15)),
    "softprob-3": ("multi", 3, dict(objective="multi:softprob", num_class=3, max_depth=4), {}),
    "forest-3": ("reg", 1, dict(objective="reg:squarederror", max_depth=4, num_parallel_tree=3, eta=0.5), {}),
    "lossguide-24": ("reg", 1, dict(objective="reg:squarederror", grow_policy="lossguide", max_leaves=24, max_depth=0), {}),
    "depth8-wide": ("reg", 1, dict(objective="reg:squarederror", max_depth=8), dict(F=120)),
}


def _identity_data(xgb, kind, K, opts):
    X, y = synth(6000, opts.get("F", 16), 11, kind, K=K, missing_frac=opts.get("missing_frac", 0.0))
    w = np.random.default_rng(3).uniform(0.5, 2.0, len(y)).astype(np.float32) if opts.get("weights") else None
    return X, y, xgb.DMatrix(X, label=y, weight=w)


@pytest.mark.parametrize("case", sorted(IDENTITY))
def test_refresh_on_the_training_data_is_the_identity(xgb, tmp_path, case):
    kind, K, params, opts = IDENTITY[case]
    params = dict(params, eta=params.get("eta", 0.3), max_bin=256)
    X, y, d = _identity_data(xgb, kind, K, opts)
    rounds = 5
    bst = xgb.Booster(params, [d])
    for i in range(rounds):
        bst.update(d, i)
    be = xgb.get_backend()
    trained = _export(xgb, bst)
    cache = be.booster_cached_margin(bst.handle, d.handle, K)
    pred = bst.predict(d, output_margin=True)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    # the same Booster, switched to update mode
    bst.set_param(_update_params({}))
    for i in range(rounds):
        bst.update(d, i)
    _assert_models_equal(_export(xgb, bst), trained)
    np.testing.assert_array_equal(be.booster_cached_margin(bst.handle, d.handle, K), cache)
    np.testing.assert_array_equal(bst.predict(d, output_margin=True), pred)
    # a model file through xgb.train(xgb_model=...): the file carries no bins (split_bin = -1)
    res = {}
    up = xgb.train(_update_params(params), d, num_boost_round=rounds, xgb_model=path, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    _assert_models_equal(_export(xgb, up), trained, tuple(k for k in R.FIELDS if k != "split_bin") + ("tree_offset", "tree_info"))
    np.testing.assert_array_equal(up.predict(d, output_margin=True), pred)


def _sums_array(sums):
    return np.concatenate([np.stack([G, H], axis=1) for G, H in sums])


_JSON_TREE = (("left_children", "left", int), ("right_children", "right", int), ("parents", "parent", int),
              ("split_indices", "split_index", int), ("split_conditions", "split_cond", float), ("default_left", "default_left", int),
              ("base_weights", "base_weight", float), ("loss_changes", "loss_chg", float), ("sum_hessian", "sum_hess", float))


def _with_trees(doc, trees):
    """A copy of the JSON model document `doc` whose trees are the restatement-form trees `trees`."""
    import copy
    doc = copy.deepcopy(doc)
    tj = doc["learner"]["gradient_booster"]["model"]["trees"]
    assert len(tj) == len(trees)
    for t, tr in zip(tj, trees):
        for jk, k, conv in _JSON_TREE:
            t[jk] = [conv(v) for v in tr[k]]
        t["split_type"] = [0] * len(tr["left"])
        t["tree_param"]["num_nodes"] = str(len(tr["left"]))
    return doc


def _load_doc(xgb, doc):
    import json
    return xgb.Booster(model_file=bytearray(json.dumps(doc).encode()))


def _scrambled(tree):
    """The same tree with its nodes in depth-first order (a left child's sibling comes after the left child's whole subtree, so
    siblings are not adjacent) and an unreachable zero leaf, like one of upstream's deleted slots, right after the root."""
    order = []
    stack = [0]
    while stack:
        i = stack.pop()
        order.append(i)
        if tree["left"][i] != -1:
            stack += [tree["right"][i], tree["left"][i]]
    new = {old: (0 if j == 0 else j + 1) for j, old in enumerate(order)}
    nn = len(order) + 1
    out = {k: np.zeros(nn, tree[k].dtype) for k in R.FIELDS}
    out["left"][:] = -1
    out["right"][:] = -1
    out["parent"][1] = 2147483647
    for old, j in new.items():
        for k in R.FIELDS:
            out[k][j] = tree[k][old]
        for k in ("left", "right"):
            out[k][j] = -1 if tree[k][old] == -1 else new[tree[k][old]]
        out["parent"][j] = tree["parent"][0] if old == 0 else new[int(tree["parent"][old])]
    return out


def _gradient_fn(xgb, params, d):
    helper = xgb.Booster({k: v for k, v in params.items() if k in ("objective", "num_class")})
    return lambda margin, r: xgb.get_backend().booster_compute_gradient(helper.handle, d.handle, margin, r)


@pytest.mark.parametrize("refresh_leaf", [0, 1])
@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic"])
def test_refresh_on_new_data_matches_the_restatement(xgb, objective, refresh_leaf):
    kind = "bin" if objective.startswith("binary") else "reg"
    params = dict(objective=objective, max_depth=5, eta=0.3, base_score=0.5, max_bin=256)
    XA, yA = synth(5000, 10, 1, kind, missing_frac=0.1)
    XB, yB = synth(4000, 10, 2, kind, missing_frac=0.1)
    dA, dB = xgb.DMatrix(XA, label=yA), xgb.DMatrix(XB, label=yB)
    trained = xgb.train(params, dA, num_boost_round=4, verbose_eval=False)
    m = _export(xgb, trained)
    up = xgb.Booster(_update_params(params, refresh_leaf=refresh_leaf), [dB], model_file=trained)
    for i in range(4):
        up.update(dB, i)
    got = _export(xgb, up)
    base = 0.0 if kind == "bin" else 0.5                       # the margin of base_score 0.5: logit(0.5) = 0 under the logistic link
    trees, sums, _ = R.update_model(m, XB, _gradient_fn(xgb, params, dB), R.Param(eta=0.3, max_depth=5), ["refresh"], refresh_leaf, 1, 1, base)
    ref = R.flatten(trees)
    _assert_models_equal(got, ref, R.FIELDS + ("tree_offset",))
    # every node's exact int64 sums, in the node order of the trees before the update
    np.testing.assert_array_equal(xgb.get_backend().booster_refresh_sums(up.handle), _sums_array(sums))
    if not refresh_leaf:
        leaf = m["left"] == -1
        np.testing.assert_array_equal(got["split_cond"][leaf], m["split_cond"][leaf])
    assert not np.array_equal(got["sum_hess"], m["sum_hess"])


def test_refresh_and_prune_match_the_restatement(xgb, tmp_path):
    params = dict(objective="reg:squarederror", max_depth=6, eta=0.3, base_score=0.5, max_bin=256)
    XA, yA = synth(6000, 12, 5, "reg")
    XB, yB = synth(5000, 12, 6, "reg")
    dA, dB = xgb.DMatrix(XA, label=yA), xgb.DMatrix(XB, label=yB)
    trained = xgb.train(params, dA, num_boost_round=4, verbose_eval=False)
    m = _export(xgb, trained)
    uparams = _update_params(dict(params, gamma=2.0, max_depth=4), updater=["refresh", "prune"], refresh_leaf=1)
    up = xgb.train(uparams, dB, num_boost_round=4, xgb_model=trained, verbose_eval=False)
    got = _export(xgb, up)
    p = R.Param(eta=0.3, gamma=2.0, max_depth=4)
    trees, _, _ = R.update_model(m, XB, _gradient_fn(xgb, params, dB), p, ["refresh", "prune"], 1, 1, 1, 0.5)
    ref = R.flatten(trees)
    _assert_models_equal(got, ref, R.FIELDS + ("tree_offset",))
    assert len(got["left"]) < len(m["left"])
    for tr in trees:                                           # no split the rule would prune is left
        _, depth, _ = R._parents_depths(tr)
        for i in np.nonzero(tr["left"] != -1)[0]:
            assert not R.prunable(tr, i, depth[i] + 1, p)
    # the compacted model serves like the restatement's
    margin = R.predict_margin(trees, [0] * len(trees), XB, 1, 0.5)[:, 0]
    np.testing.assert_array_equal(up.predict(dB, output_margin=True), margin)
    leaves = up.predict(dB, pred_leaf=True).astype(np.int64).reshape(len(yB), -1)
    for t, tr in enumerate(trees):
        np.testing.assert_array_equal(leaves[:, t], R.leaf_of(tr, XB))
    contribs = up.predict(dB, pred_contribs=True)
    np.testing.assert_allclose(contribs.sum(axis=1), margin, rtol=0, atol=1e-4)
    import json
    path = str(tmp_path / "doc.json")
    up.save_model(path)
    ref_bst = _load_doc(xgb, _with_trees(json.load(open(path)), trees))      # the restatement's model, served by the engine
    np.testing.assert_array_equal(contribs, ref_bst.predict(dB, pred_contribs=True))
    np.testing.assert_array_equal(up.predict(dB, pred_leaf=True), ref_bst.predict(dB, pred_leaf=True))
    for fmt in ("json", "ubj"):
        path = str(tmp_path / ("m." + fmt))
        up.save_model(path)
        np.testing.assert_array_equal(xgb.Booster(model_file=path).predict(dB, output_margin=True), margin)
    np.testing.assert_array_equal(pickle.loads(pickle.dumps(up)).predict(dB, output_margin=True), margin)


@pytest.mark.parametrize("objective", ["reg:squarederror", "multi:softprob"])
def test_refresh_and_prune_of_a_model_with_deleted_slots_and_non_adjacent_children(xgb, tmp_path, objective):
    """Upstream models may keep deleted node slots (zero leaves no path reaches) and allocate children apart: the refresh leaves
    the unreachable slots out, the compaction drops them, and the result serves through the predictor's general path."""
    import json
    K = 3 if objective == "multi:softprob" else 1
    kind = "multi" if K > 1 else "reg"
    params = dict(objective=objective, max_depth=5, eta=0.3, base_score=0.5, max_bin=256, **({"num_class": K} if K > 1 else {}))
    XA, yA = synth(5000, 10, 31, kind, K=K, missing_frac=0.1)
    XB, yB = synth(4000, 10, 32, kind, K=K, missing_frac=0.1)
    dA, dB = xgb.DMatrix(XA, label=yA), xgb.DMatrix(XB, label=yB)
    trained = xgb.train(params, dA, num_boost_round=3, verbose_eval=False)
    path = str(tmp_path / "m.json")
    trained.save_model(path)
    m = _export(xgb, trained)
    scrambled = [_scrambled(R.tree_slice(m, t)) for t in range(len(m["tree_info"]))]
    foreign = _load_doc(xgb, _with_trees(json.load(open(path)), scrambled))
    fm = _export(xgb, foreign)
    assert any(np.any(tr["right"][tr["left"] != -1] != tr["left"][tr["left"] != -1] + 1) for tr in scrambled)
    np.testing.assert_array_equal(foreign.predict(dB, output_margin=True), trained.predict(dB, output_margin=True))
    p = R.Param(eta=0.3, gamma=1.0, max_depth=3)
    up = xgb.Booster(_update_params(dict(params, gamma=1.0, max_depth=3), updater="refresh,prune"), [dB], model_file=foreign)
    for i in range(3):
        up.update(dB, i)
    got = _export(xgb, up)
    trees, sums, _ = R.update_model(fm, XB, _gradient_fn(xgb, params, dB), p, ["refresh", "prune"], 1, K, 1, 0.5)
    _assert_models_equal(got, R.flatten(trees), tuple(k for k in R.FIELDS if k != "split_bin") + ("tree_offset",))
    np.testing.assert_array_equal(xgb.get_backend().booster_refresh_sums(up.handle), _sums_array(sums))
    assert len(got["left"]) < len(fm["left"]) - len(scrambled)                  # the dead slots and pruned nodes are gone
    margin = R.predict_margin(trees, [int(x) for x in fm["tree_info"]], XB, K, 0.5)
    np.testing.assert_array_equal(up.predict(dB, output_margin=True).reshape(len(yB), K), margin)
    leaves = up.predict(dB, pred_leaf=True).astype(np.int64).reshape(len(yB), -1)
    for t, tr in enumerate(trees):
        np.testing.assert_array_equal(leaves[:, t], R.leaf_of(tr, XB))


def test_refresh_of_the_real_xgboost_iris_model(xgb):
    from sklearn.datasets import load_iris
    from test_iris_real_xgboost_pin import GOLD, PARAMS, _reference_model
    X, y = load_iris(return_X_y=True)
    X, y = X.astype(np.float32), y.astype(np.float32)
    d = xgb.DMatrix(X, label=y)
    up = xgb.train(_update_params(dict(PARAMS, tree_method="hist")), d, num_boost_round=20, xgb_model=GOLD, verbose_eval=False)
    got = _export(xgb, up)
    fixture = _reference_model()
    trees, _, _ = R.update_model(fixture, X, _gradient_fn(xgb, PARAMS, d), R.Param(eta=0.3, max_depth=3), ["refresh"], 1, 3, 1, 0.5)
    _assert_models_equal(got, R.flatten(trees), tuple(k for k in R.FIELDS if k != "split_bin") + ("tree_offset",))
    # the CUDA path retrains this model tree for tree (test_iris_real_xgboost_pin.py): refreshing it keeps its statistics
    np.testing.assert_array_equal(got["left"], fixture["left"])
    np.testing.assert_allclose(got["sum_hess"], fixture["sum_hess"], rtol=1e-4, atol=1e-5)
    internal = fixture["left"] != -1
    np.testing.assert_allclose(got["loss_chg"][internal], fixture["loss_chg"][internal], rtol=1e-4, atol=1e-5)
    leaf = ~internal
    np.testing.assert_allclose(got["split_cond"][leaf], fixture["split_cond"][leaf], rtol=0, atol=1e-5)
    # the fixture's leaves hold the unscaled weight, this engine's leaves eta * weight (DESIGN.md "Refresh and prune")
    np.testing.assert_allclose(got["base_weight"][leaf], np.float32(0.3) * fixture["base_weight"][leaf], rtol=1e-4, atol=1e-5)


def test_evaluation_and_early_stopping_in_update_mode(xgb):
    params = dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256)
    XA, yA = synth(5000, 10, 7, "reg")
    XB, yB = synth(4000, 10, 8, "reg")
    XV, yV = synth(3000, 10, 9, "reg")
    dA, dB, dV = xgb.DMatrix(XA, label=yA), xgb.DMatrix(XB, label=yB), xgb.DMatrix(XV, label=yV)
    trained = xgb.train(params, dA, num_boost_round=6, verbose_eval=False)
    res = {}
    up = xgb.train(_update_params(params), dB, num_boost_round=6, xgb_model=trained, evals=[(dB, "train"), (dV, "valid")], evals_result=res, verbose_eval=False)
    for r in range(6):
        pred = up[: r + 1].predict(dV)
        rmse = float(np.sqrt(np.mean((pred.astype(np.float64) - yV) ** 2)))
        assert abs(res["valid"]["rmse"][r] - rmse) < 1e-5
    # early stopping: each refreshed layer is a Newton step on dB's own squared error, so its training rmse falls every round;
    # told to maximize it, early stopping with patience 1 must stop after the second round
    res = {}
    up = xgb.train(_update_params(params), dB, num_boost_round=6, xgb_model=trained, evals=[(dB, "train")], evals_result=res,
                   early_stopping_rounds=1, maximize=True, verbose_eval=False)
    hist = res["train"]["rmse"]
    assert len(hist) == 2 and hist[1] < hist[0]
    assert up.num_boosted_rounds() == 2
    assert up.best_iteration == 6 + 0          # upstream's numbering: the rounds of the xgb_model first, then this run's


def test_update_mode_errors(xgb):
    params = dict(objective="reg:squarederror", max_depth=3, max_bin=256)
    X, y = synth(2000, 6, 1, "reg")
    d = xgb.DMatrix(X, label=y)
    trained = xgb.train(params, d, num_boost_round=2, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="cannot exceed the previous training rounds"):
        xgb.train(_update_params(params), d, num_boost_round=3, xgb_model=trained, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="dart"):
        xgb.train(_update_params(dict(params, booster="dart")), d, num_boost_round=1, xgb_model=trained, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="updater"):
        xgb.train(_update_params(params, updater="refresh,grow_quantile_histmaker"), d, num_boost_round=1, xgb_model=trained, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="updater"):
        xgb.train(dict(params, process_type="update"), d, num_boost_round=1, xgb_model=trained, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError, match="process_type"):
        xgb.train(dict(params, process_type="refresh"), d, num_boost_round=1, verbose_eval=False)


def test_default_mode_ignores_updater_and_refresh_leaf(xgb):
    params = dict(objective="reg:squarederror", max_depth=4, max_bin=256)
    X, y = synth(3000, 8, 2, "reg")
    d = xgb.DMatrix(X, label=y)
    a = xgb.train(params, d, num_boost_round=3, verbose_eval=False)
    b = xgb.train(dict(params, process_type="default", updater="grow_quantile_histmaker,prune", refresh_leaf=0), d, num_boost_round=3, verbose_eval=False)
    _assert_models_equal(_export(xgb, a), _export(xgb, b))
    assert a.save_config() == b.save_config()


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_gpu_refresh_equals_single_gpu(xgb, tmp_path):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    n, F = 40000, 12
    params = dict(objective="binary:logistic", max_depth=5, eta=0.3, max_bin=256)
    XA, yA = synth(n, F, 21, "bin")
    model = str(tmp_path / "base.ubj")
    xgb.train(params, xgb.DMatrix(XA, label=yA), num_boost_round=4, verbose_eval=False).save_model(model)
    out = str(tmp_path / "refreshed.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29613", os.path.join(ROOT, "tests", "helpers", "refresh_shard_worker.py"), model, out, str(n), str(F)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    XB, yB = synth(n, F, 22, "bin")
    single = xgb.train(_update_params(params, updater="refresh,prune", gamma=1.0), xgb.DMatrix(XB, label=yB), num_boost_round=4, xgb_model=model,
                       verbose_eval=False)
    _assert_models_equal(_export(xgb, xgb.Booster(model_file=out)), _export(xgb, single), tuple(k for k in R.FIELDS if k != "split_bin") + ("tree_offset",))
