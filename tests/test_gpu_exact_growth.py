"""Whole trees bit for bit against the oracle trained on the device's fixed-point grid (Trainer.set_device_grid): for
objectives whose gradients are plain IEEE arithmetic on both sides (reg:squarederror, weighted or not, and binary:hinge),
every exported array, the trainer's prediction cache and predict(output_margin=True) must equal the oracle's as bits after
every round.  No tolerance: any difference in split arithmetic, tie order, expansion or cache update shows."""
import numpy as np
import pytest

from util import synth

pytestmark = pytest.mark.gpu

ARRAYS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def grow_and_compare(xgb, oracle, X, y, params, rounds, weights=None):
    n = X.shape[0]
    params = dict(tree_method="hist", max_bin=256, **params)
    d = xgb.DMatrix(X, label=y, weight=weights)
    bst = xgb.Booster(params, [d])
    cuts = _be().dmatrix_get_cuts(d.handle, 256)
    bins = _be().dmatrix_get_bins(d.handle, 256)
    ref = oracle.Trainer(params, bins=bins, cuts=cuts, y=y, weights=weights, base_score=params["base_score"])
    ref.set_device_grid(n)
    for r in range(rounds):
        bst.update(d, r)
        ref.update()
        m, mr = _be().booster_export_model(bst.handle), ref.model()
        np.testing.assert_array_equal(m["tree_offset"], mr["tree_offset"], err_msg="round %d: tree sizes" % r)
        for k in ARRAYS:
            a, b = (m[k], mr[k]) if m[k].dtype != np.float32 else (_u32(m[k]), _u32(mr[k]))
            np.testing.assert_array_equal(a, b, err_msg="round %d: %s" % (r, k))
        np.testing.assert_array_equal(_u32(_be().booster_cached_margin(bst.handle, d.handle, 1)), _u32(ref.margins()), err_msg="round %d: cache" % r)
    margin = bst.predict(d, output_margin=True).reshape(n, 1)
    np.testing.assert_array_equal(_u32(margin), _u32(oracle.predict_margin(mr, X)))
    return m


def _nondyadic_weights(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.integers(1, 30, n) / 7.0).astype(np.float32)


CASES = {
    "sqerr-F28-depth6": (20000, 28, "reg", 0.0, dict(objective="reg:squarederror", max_depth=6, eta=0.3), 4, False),
    "sqerr-weighted-F100": (20000, 100, "reg", 0.0, dict(objective="reg:squarederror", max_depth=5, eta=0.3), 3, True),
    "hinge-F104-missing": (15000, 104, "bin", 0.1, dict(objective="binary:hinge", max_depth=5, eta=0.3), 3, False),
    "lossguide-F41": (20000, 41, "reg", 0.05, dict(objective="reg:squarederror", grow_policy="lossguide", max_leaves=24, max_depth=0, eta=0.3), 3, False),
    "monotone-mds-alpha": (15000, 12, "reg", 0.0, dict(objective="reg:squarederror", max_depth=5, eta=0.3, alpha=0.5, max_delta_step=0.6,
                                                      monotone_constraints="(1,-1,0,1,0,0,-1,0,0,0,1,0)"), 4, False),
    "gamma-mcw": (8000, 20, "reg", 0.0, dict(objective="reg:squarederror", max_depth=6, eta=0.3, gamma=2.0, min_child_weight=40), 4, True),
    "subsample-bynode": (20000, 30, "bin", 0.0, dict(objective="binary:hinge", max_depth=5, eta=0.3, subsample=0.8, colsample_bynode=0.5, seed=3), 3, False),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_trees_bit_exact_on_the_device_grid(xgb, oracle, case):
    n, F, kind, missing, hp, rounds, weighted = CASES[case]
    X, y = synth(n, F, 41, kind, missing_frac=missing)
    w = _nondyadic_weights(n, 5) if weighted else None
    grow_and_compare(xgb, oracle, X, y, dict(base_score=0.25, **hp), rounds, weights=w)


def test_duplicated_and_negated_columns(xgb, oracle):
    """Exact ties across features (a copy) and across directions (a negated copy)."""
    X, y = synth(12000, 10, 43, "reg")
    X = np.ascontiguousarray(np.concatenate([X, X[:, :4], -X[:, :4]], axis=1))
    grow_and_compare(xgb, oracle, X, y, dict(objective="reg:squarederror", max_depth=6, eta=0.3, base_score=0.0), 3)


def test_large_matrix_on_the_18_bit_grid(xgb, oracle):
    """1.2 M rows: the 18-bit grid and the histogram kernels' overflow windows."""
    X, y = synth(1_200_000, 28, 47, "reg")
    grow_and_compare(xgb, oracle, X, y, dict(objective="reg:squarederror", max_depth=6, eta=0.3, base_score=0.5), 2)


def test_wide_matrix_splits_above_feature_32767(xgb, oracle):
    """F = 33 000 with the informative features at f >= 32 768, with missing values: the prediction cache must read the
    right column and send missing values the learned way."""
    rng = np.random.default_rng(49)
    n, F = 1500, 33000
    X = rng.integers(0, 16, size=(n, F)).astype(np.float32)
    informative = [32768, 32900, 32999]
    y = (X[:, informative] @ np.array([1.0, -0.7, 0.4], np.float32) + 0.1 * rng.standard_normal(n)).astype(np.float32)
    for f in informative:
        X[rng.random(n) < 0.2, f] = np.nan
    m = grow_and_compare(xgb, oracle, X, y, dict(objective="reg:squarederror", max_depth=3, eta=0.5, base_score=0.0), 3)
    assert (m["split_index"][m["tree_offset"][:-1]] >= 32768).all()        # every root splits above 32 767
