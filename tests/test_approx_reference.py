"""tree_method=approx restated on the CPU (tests/approx_reference.py): each tree's cuts are the shared cut rule with its
hessian as the weights, bit for bit; constant-hessian objectives grow hist trees; the Python layer stops warning."""
import warnings

import numpy as np
import pytest

import approx_reference as AR
import cuts_reference as CR
import forest_reference as FR
from util import synth


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_cuts(a, b):
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(_u32(a[1]), _u32(b[1]))
    np.testing.assert_array_equal(_u32(a[2]), _u32(b[2]))


@pytest.mark.parametrize("objective,kind,K", [("binary:logistic", "bin", 1), ("multi:softprob", "multi", 3), ("count:poisson", "count", 1),
                                              ("reg:pseudohubererror", "reg", 1)])
def test_tree_cuts_are_the_cut_rule_with_the_hessian(oracle, objective, kind, K):
    X, y = synth(3000, 6, 3, kind, K=K, quantised=False, missing_frac=0.05)
    X[:, 5] = np.round(X[:, 5] * 4) + np.float32(0)       # a feature with fewer distinct values than bins keeps its cuts
    w = np.random.default_rng(1).uniform(0.5, 2.0, len(y)).astype(np.float32)
    params = dict(objective=objective, max_bin=64, num_class=K) if K > 1 else dict(objective=objective, max_bin=64)
    margin = np.random.default_rng(2).standard_normal((len(y), K)).astype(np.float32) * 0.5
    gp = oracle.gradient(params, margin, y, w)
    for k in range(K):
        h = gp[:, k, 1]
        assert CR.in_exact_regime(h)
        got = AR.tree_cuts(X, 64, h)
        ref = CR.make_cuts(X, 64, h)
        _same_cuts(got, ref)
        assert got[3] == ref[3]
    # the hessian moves the cuts of the wide features and no others
    own = CR.make_cuts(X, 64, w)
    hc = CR.make_cuts(X, 64, gp[:, 0, 1])
    cut = lambda c, f: c[1][c[0][f]:c[0][f + 1]]     # noqa: E731
    assert all(not np.array_equal(cut(own, f), cut(hc, f)) for f in range(5))
    np.testing.assert_array_equal(cut(own, 5), cut(hc, 5))


def test_zero_total_weight(oracle):
    """Every hessian 0 (a saturated logistic): every target is 0, met by the first run, so a wide feature's cuts are its second
    distinct value and the end cut."""
    X, _ = synth(2000, 3, 4, quantised=False)
    h = np.zeros(len(X), np.float32)
    got = AR.tree_cuts(X, 32, h)
    _same_cuts(got, CR.make_cuts(X, 32, h))
    for f in range(3):
        d = np.unique(X[:, f])
        np.testing.assert_array_equal(_u32(got[1][got[0][f]:got[0][f + 1]]), _u32([d[1], CR.end_cut(d[-1])]))


@pytest.mark.parametrize("objective", ["reg:squarederror"])
def test_constant_hessian_grows_hist_trees(oracle, objective):
    X, y = synth(2000, 5, 5, "reg", quantised=False)
    w = np.random.default_rng(3).uniform(0.5, 2.0, len(y)).astype(np.float32)
    params = dict(objective=objective, max_bin=32, max_depth=4, eta=0.5, base_score=0.5)
    a = AR.ApproxTrainer(params, X, y, weights=w, base_score=0.5)
    b = FR.ForestTrainer(params, X, y, 1, weights=w, base_score=0.5)
    for _ in range(3):
        a.update()
        b.update()
    for k in FR.KEYS:
        np.testing.assert_array_equal(a.model()[k], b.model()[k], err_msg=k)


@pytest.mark.parametrize("objective,kind,K,P", [("binary:logistic", "bin", 1, 1), ("multi:softprob", "multi", 3, 1), ("binary:logistic", "bin", 1, 2)])
def test_each_tree_grows_on_its_hessian_cuts(oracle, objective, kind, K, P):
    X, y = synth(2000, 5, 6, kind, K=K, quantised=False, missing_frac=0.03)
    params = dict(objective=objective, max_bin=32, max_depth=4, eta=0.5, base_score=0.5, subsample=0.8 if P > 1 else 1.0, seed=3)
    if K > 1:
        params["num_class"] = K
    t = AR.ApproxTrainer(params, X, y, P=P, base_score=0.5)
    for r in range(3):
        pre = t.margins()
        t.update()
        gp = oracle.gradient(params, pre, y)
        for k in range(K):
            for j in range(P):
                _same_cuts(t.tree_cuts[t.indptr[r] + k * P + j], CR.make_cuts(X, 32, gp[:, k, 1]))
    # the trees split on thresholds of their own cuts
    m = t.model()
    for i in range(len(t.trees)):
        a, b = int(m["tree_offset"][i]), int(m["tree_offset"][i + 1])
        ptrs, vals = t.tree_cuts[i][0], t.tree_cuts[i][1]
        for node in range(a, b):
            if m["left"][node] != -1:
                f = m["split_index"][node]
                assert m["split_cond"][node] in vals[ptrs[f]:ptrs[f + 1]]


def test_python_layer_applies_approx_and_warns_for_exact():
    from sagemaker_xgboost_container_b200 import core
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert core._check_unapplied("tree_method", "approx") == "approx"
    with pytest.warns(UserWarning, match="tree_method=exact"):
        core._check_unapplied("tree_method", "exact")
