"""Routed depth-wise growth (run with `pytest -m gpu` on an H100): trees up to max_depth 7 keep one node id per row and write
only the built children's rows per level; deeper trees and lossguide move every row of a split node through part_kernel.
Structure must equal the oracle's exactly (leaves within 1e-5) across tile boundaries, tail widths, missing values, nodes
that stop splitting early, sampling, several classes, dart and forests, and the prediction cache, whose walk starts at the
node each row was routed to, must equal predict() bit for bit."""
import numpy as np
import pytest

import dart_reference as DR
import forest_reference as FR
from util import assert_same_structure, first_structural_difference, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
LEAF_TOL = 1e-5
MARGIN_TOL = 2e-5
TILE = 2048           # rows per route / scatter tile (tree.h kRouteTile)


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _train_check(xgb, oracle, X, y, params, rounds):
    """Trains on the device and in the oracle; returns the device model after the checks every case shares."""
    K = int(params.get("num_class", 1))
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    ref = oracle.train(params, X, y, rounds)
    mr = ref.model()
    assert first_structural_difference(m, mr) is None, "tree structure differs first at tree %s" % first_structural_difference(m, mr)
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    cache = _be().booster_cached_margin(bst.handle, d.handle, K)
    np.testing.assert_allclose(cache, ref.margins(), rtol=0, atol=MARGIN_TOL)
    np.testing.assert_array_equal(_u32(cache), _u32(bst.predict(d, output_margin=True).reshape(-1, K)))
    return m


def _depth_of_nodes(m, t):
    a, b = int(m["tree_offset"][t]), int(m["tree_offset"][t + 1])
    parent = m["parent"][a:b]
    depth = np.zeros(b - a, np.int32)
    for i in range(1, b - a):
        depth[i] = depth[parent[i]] + 1
    return depth, m["left"][a:b] == -1


@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, 2 * TILE + 37])
def test_rows_around_one_tile(xgb, oracle, n):
    X, y = synth(n, 28, 61, "reg")
    _train_check(xgb, oracle, X, y, dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3), 6)


# tail widths 0 (F = 8: one padded group), 4 (F = 36, 100: by position through the scatter), 8 (F = 104: the aligned line)
@pytest.mark.parametrize("F", [8, 36, 100, 104])
@pytest.mark.parametrize("objective,kind", [("reg:squarederror", "reg"), ("binary:logistic", "bin")])
def test_tail_widths(xgb, oracle, F, objective, kind):
    X, y = synth(20000, F, 62 + F, kind)
    _train_check(xgb, oracle, X, y, dict(objective=objective, tree_method="hist", max_bin=256, max_depth=6, eta=0.3), 4)


@pytest.mark.parametrize("F", [36, 104])
def test_missing_values_both_default_directions(xgb, oracle, F):
    X, y = synth(30000, F, 63, "reg", quantised=False, missing_frac=0.1)
    # missing in feature 0 behaves like a large value, in feature 1 like a small one: both default directions are learnt
    y = (y + np.nan_to_num(X[:, 0], nan=3.0) - np.nan_to_num(X[:, 1], nan=3.0)).astype(np.float32)
    m = _train_check(xgb, oracle, X, y, dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3), 5)
    internal = m["left"] != -1
    assert set(np.unique(m["default_left"][internal])) == {0, 1}


@pytest.mark.parametrize("hp", [dict(gamma=40.0), dict(min_child_weight=600)])
def test_nodes_that_stop_splitting_early(xgb, oracle, hp):
    """Rows of a node that becomes a leaf at levels 1-3 keep its id while the rest of the tree goes on splitting."""
    X, y = synth(3 * TILE + 5, 20, 64, "reg")
    y = (y + 4.0 * (X[:, 0] > 1.5)).astype(np.float32)
    m = _train_check(xgb, oracle, X, y, dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3, **hp), 5)
    early = False
    for t in range(len(m["tree_info"])):
        depth, leaf = _depth_of_nodes(m, t)
        early |= bool((leaf & (depth >= 1) & (depth <= 3)).any()) and bool((depth >= 4).any())
    assert early, "some tree should park rows at levels 1-3 and still grow deeper elsewhere"


@pytest.mark.parametrize("objective,kind,K,hp", [
    ("reg:squarederror", "reg", 1, dict(subsample=0.7, seed=3)),
    ("multi:softprob", "multi", 3, dict()),
    ("binary:logistic", "bin", 1, dict(subsample=0.8, colsample_bynode=0.7, seed=4)),
])
def test_sampling_and_classes(xgb, oracle, objective, kind, K, hp):
    X, y = synth(2 * TILE + 100, 24, 65, kind, K=K)
    params = dict(objective=objective, tree_method="hist", max_bin=256, max_depth=6, eta=0.3, **hp)
    if K > 1:
        params["num_class"] = K
    _train_check(xgb, oracle, X, y, params, 4)


@pytest.mark.parametrize("depth", [1, 6, 7, 8])
def test_depths_of_both_paths(xgb, oracle, depth):
    """max_depth 1, 6 and 7 are routed, 8 goes through part_kernel: each equals the oracle on the same data."""
    X, y = synth(3 * TILE + 11, 30, 66, "reg")
    m = _train_check(xgb, oracle, X, y, dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=depth, eta=0.3), 4)
    assert max(_depth_of_nodes(m, t)[0].max() for t in range(len(m["tree_info"]))) == depth


def test_routed_and_moved_rows_give_the_same_trees(xgb):
    """Trees that never reach depth 6 (min_child_weight allows at most 6 leaves) are the same model at max_depth 6, 7 (routed)
    and 8 (part_kernel), every array and the prediction cache bit for bit."""
    n = 2 * TILE + 300
    X, y = synth(n, 30, 67, "reg")
    out = []
    for depth in (6, 7, 8):
        params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=depth, eta=0.3, min_child_weight=n // 7)
        d = xgb.DMatrix(X, label=y)
        bst = xgb.train(params, d, num_boost_round=5, verbose_eval=False)
        m = _be().booster_export_model(bst.handle)
        m["cache"] = _be().booster_cached_margin(bst.handle, d.handle, 1)
        out.append(m)
    assert max(_depth_of_nodes(out[0], t)[0].max() for t in range(len(out[0]["tree_info"]))) >= 3
    for m in out[1:]:
        for k in ("tree_offset", "left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight",
                  "loss_chg", "sum_hess", "cache"):
            a, b = np.asarray(out[0][k]), np.asarray(m[k])
            np.testing.assert_array_equal(_u32(a) if a.dtype == np.float32 else a, _u32(b) if b.dtype == np.float32 else b, err_msg=k)


def test_dart(xgb, oracle):
    X, y = synth(TILE + 3, 20, 68, "reg")
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3, base_score=0.5, seed=7,
                  booster="dart", rate_drop=0.3, one_drop=1)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    t = oracle.Trainer(params, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256), y=y,
                       base_score=params["base_score"])
    t.set_device_grid(X.shape[0])
    ref = DR.DartTrainer(params, X, trainer=t)
    for r in range(8):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    np.testing.assert_array_equal(_u32(_be().booster_cached_margin(bst.handle, d.handle, 1)), _u32(ref.m_full))


def test_forest(xgb):
    X, y = synth(2 * TILE + 9, 16, 69, "reg")
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.7, base_score=0.5, seed=5,
                  num_parallel_tree=3, subsample=0.8)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(params, [d])
    ref = FR.ForestTrainer(params, X, y, 3, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256),
                           base_score=0.5)
    for r in range(3):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    cache = _be().booster_cached_margin(bst.handle, d.handle, 1)
    np.testing.assert_array_equal(_u32(cache), _u32(ref.margins()))
    np.testing.assert_array_equal(_u32(cache), _u32(bst.predict(d, output_margin=True).reshape(-1, 1)))
