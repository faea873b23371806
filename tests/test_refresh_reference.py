"""The NumPy restatement of process_type=update (tests/refresh_reference.py) on CPU: refreshing an oracle-trained model on its
own data gives the model back (to the oracle's double-precision sums vs the fixed-point grid), its prune equals a brute-force
bottom-up prune, and the compaction keeps every prediction."""
import numpy as np
import pytest

import refresh_reference as R
from util import synth

PARAMS = dict(objective="reg:squarederror", max_depth=5, eta=0.3, base_score=0.5, max_bin=256)


def _sqerr(y):
    return lambda m, r: np.stack([m[:, 0] - y, np.ones_like(y)], -1)[:, None, :].astype(np.float32)


def test_refresh_of_an_oracle_model_on_its_own_data_is_the_identity(oracle):
    X, y = synth(3000, 12, 3, "reg", missing_frac=0.1)
    m = oracle.train(PARAMS, X, y, 4).model()
    trees, _, _ = R.update_model(m, X, _sqerr(y), R.Param(eta=0.3, max_depth=5), ["refresh"], 1, 1, 1, 0.5)
    f = R.flatten(trees)
    for k in ("left", "right", "parent", "split_index", "default_left", "sum_hess"):
        np.testing.assert_array_equal(f[k], m[k], err_msg=k)
    for k in ("split_cond", "base_weight", "loss_chg"):
        np.testing.assert_allclose(f[k], m[k], rtol=2e-5, atol=1e-6, err_msg=k)


def _brute_prune(tree, p):
    """Repeat until nothing changes: any split of two leaves that the rule prunes becomes a leaf (children removed)."""
    tree = {k: v.copy() for k, v in tree.items()}
    par, depth, alive = R._parents_depths(tree)
    changed = True
    while changed:
        changed = False
        for pid in range(len(tree["left"]) - 1, -1, -1):
            if alive[pid] and tree["left"][pid] != -1 and R.prunable(tree, pid, depth[pid] + 1, p):
                alive[tree["left"][pid]] = alive[tree["right"][pid]] = False
                R.make_leaf(tree, pid, p)
                changed = True
    return R.compact(tree, alive)


@pytest.mark.parametrize("gamma,max_depth", [(5.0, 5), (0.0, 3), (40.0, 2)])
def test_prune_equals_a_brute_force_bottom_up_prune(oracle, gamma, max_depth):
    X, y = synth(3000, 12, 4, "reg")
    m = oracle.train(dict(PARAMS, max_depth=6), X, y, 3).model()
    p = R.Param(eta=0.3, gamma=gamma, max_depth=max_depth)
    for t in range(3):
        tree = R.tree_slice(m, t)
        got, _, _ = R.update_tree(tree, X, np.zeros(len(y), np.int64), np.zeros(len(y), np.int64), np.float32(1), np.float32(1), p, ["prune"], 1)
        ref = _brute_prune(tree, p)
        for k in R.FIELDS:
            np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
        assert len(got["left"]) < len(tree["left"])
        _, depth, _ = R._parents_depths(got)
        for i in np.nonzero(got["left"] != -1)[0]:              # nothing the rule would prune is left
            assert not R.prunable(got, i, depth[i] + 1, p)


def test_compaction_keeps_predictions(oracle):
    X, y = synth(2000, 10, 5, "reg", missing_frac=0.2)
    m = oracle.train(dict(PARAMS, max_depth=6), X, y, 2).model()
    tree = R.tree_slice(m, 1)
    alive = np.ones(len(tree["left"]), bool)
    R.prune(tree, R.Param(eta=0.3, max_depth=3), alive)          # prunes everything below depth 3
    assert not alive.all()
    comp = R.compact(tree, alive)
    assert np.all(comp["left"][comp["left"] != -1] > np.nonzero(comp["left"] != -1)[0])      # children after parents
    internal = comp["left"] != -1
    np.testing.assert_array_equal(comp["right"][internal], comp["left"][internal] + 1)        # sibling pairs stay adjacent
    np.testing.assert_array_equal(comp["split_cond"][R.leaf_of(comp, X)], tree["split_cond"][R.leaf_of(tree, X)])
