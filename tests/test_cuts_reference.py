"""CPU checks of tests/cuts_reference.py, the exact restatement of the quantile cuts: against the oracle (oracle.make_cuts /
oracle.bin_matrix) on random data inside the exact regime, and against answers worked out by hand for the edges (the
list / quantile boundary with and without missing values, +-inf, +-0, denormals, FLT_MAX, all-missing, constant and
one-row columns) and for the multi-GPU summary and merge.

The oracle is compared with `==`: its qsort may pick -0.0 as the zero run's representative.  The restatement is compared
bit for bit."""
import numpy as np
import pytest

import cuts_reference as R

F32 = np.float32
FLT_MAX = np.finfo(np.float32).max
TINY = np.float32(2.0 ** -149)


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def assert_bitwise(got, want):
    np.testing.assert_array_equal(bits(got), bits(np.asarray(want, np.float32)))


def _data(rng, n, F, kind, missing_frac):
    X = rng.standard_normal((n, F)).astype(np.float32)
    if kind == "list":                        # at most 48 distinct values per feature: the list branch for max_bin >= 48
        X = (np.round(np.clip(X, -3, 3) * 8) / 8).astype(np.float32)
    else:                                     # long duplicate runs next to singletons
        X[:, 0] = np.round(X[:, 0] * 4) / 4
        X[rng.random(n) < 0.6, 1] = 0.0
    if missing_frac:
        X[rng.random((n, F)) < missing_frac] = np.nan
    return X


@pytest.mark.parametrize("kind,max_bin", [("list", 64), ("list", 256), ("quantile", 2), ("quantile", 16), ("quantile", 256)])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("missing_frac", [0.0, 0.05])
def test_restatement_matches_oracle(oracle, kind, max_bin, weighted, missing_frac):
    rng = np.random.default_rng(7 + max_bin)
    n, F = 6000, 5
    X = _data(rng, n, F, kind, missing_frac)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    if weighted:
        w[rng.random(n) < 0.05] = 0.0
        assert R.in_exact_regime(w)
    ptrs, vals, mins, hm = R.make_cuts(X, max_bin, w)
    optrs, ovals, omins, ohm = oracle.make_cuts(X, max_bin, w)
    assert hm == ohm == (missing_frac > 0)
    np.testing.assert_array_equal(ptrs, optrs)
    assert np.all(vals == ovals) and np.all(mins == omins)
    if kind == "quantile":
        assert ptrs[1] - ptrs[0] <= R.num_bins(max_bin, hm) and ptrs[-1] > F
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals), oracle.bin_matrix(X, optrs, ovals))


def test_exact_regime_bound():
    assert R.in_exact_regime(np.full(1000, 0.1, np.float32))
    wide = np.array([2.0 ** -20, 2.0 ** 20] * 4096, np.float32)    # 2^40 units each for the large ones, 2^12 of them
    assert not R.in_exact_regime(np.concatenate([wide, wide]))
    X = np.arange(len(wide) * 2, dtype=np.float32)[:, None]
    with pytest.raises(R.NotExact):
        R.make_cuts(X, 16, np.concatenate([wide, wide]))


def _col(values):
    return np.asarray(values, np.float32)[:, None]


@pytest.mark.parametrize("m", [15, 16, 17])
def test_list_and_quantile_boundary(oracle, m):
    """m = nb-1, nb, nb+1 distinct values 0..m-1 once each, max_bin = 16"""
    X = _col(np.arange(m))
    ptrs, vals, mins, hm = R.make_cuts(X, 16)
    if m <= 16:
        want = list(range(1, m)) + [F32(m - 1) + (F32(m - 1) + R.EPS)]
    else:       # W = 17, targets 17k/16: C_i = i + 1 first reaches it at i = k (k < 16), the cut is d[k + 1] = k + 1
        want = list(range(2, 17)) + [F32(16) + (F32(16) + R.EPS)]
    assert_bitwise(vals, want)
    assert_bitwise(mins, [-R.EPS])
    assert not hm
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals)[:, 0], np.minimum(np.searchsorted(np.array(want, np.float32), X[:, 0], "right"), len(want) - 1))
    optrs, ovals, _, _ = oracle.make_cuts(X, 16)
    assert np.all(ovals == vals)


@pytest.mark.parametrize("m,nan", [(255, True), (256, True), (256, False), (257, False)])
def test_255_vs_256_bins(oracle, m, nan):
    """a missing value anywhere leaves 255 bins: 255 distinct values still list, 256 take the quantile branch"""
    col = np.arange(m, dtype=np.float32)
    X = np.stack([col, col], 1)
    if nan:
        X[3, 1] = np.nan
    ptrs, vals, mins, hm = R.make_cuts(X, 256)
    assert hm == nan
    nb = 255 if nan else 256
    if m <= nb:
        want = list(range(1, m)) + [F32(m - 1) + (F32(m - 1) + R.EPS)]
    else:       # W = m = nb + 1: cut k = d[ceil(k m / nb)] = k + 1 for k < nb
        want = list(range(2, nb + 1)) + [F32(m - 1) + (F32(m - 1) + R.EPS)]
    assert_bitwise(vals[ptrs[0]:ptrs[1]], want)
    optrs, ovals, _, ohm = oracle.make_cuts(X, 256)
    np.testing.assert_array_equal(optrs, ptrs)
    assert ohm == hm and np.all(ovals == vals)
    b = R.bin_matrix(X, ptrs, vals)
    assert b[:, 0].max() == len(want) - 1
    if nan:        # with 255 bins no value reaches the missing code
        assert b[3, 1] == 255 and (b[:, 1] == 255).sum() == 1


@pytest.mark.parametrize("nan", [False, True])
def test_infinities_are_values(oracle, nan):
    inf = np.inf
    X = _col([1, 2, inf, -inf, 2, inf] + ([np.nan, np.nan] if nan else []))
    ptrs, vals, mins, hm = R.make_cuts(X, 256)
    assert_bitwise(vals, [1, 2, inf, inf])       # +inf is a cut, and the end cut overflows to +inf
    assert_bitwise(mins, [-inf])
    b = R.bin_matrix(X, ptrs, vals)[:, 0]
    np.testing.assert_array_equal(b, [1, 2, 3, 0, 2, 3] + ([255, 255] if nan else []))
    optrs, ovals, omins, ohm = oracle.make_cuts(X, 256)
    assert ohm == hm == nan
    assert np.all(ovals == vals) and np.all(omins == mins)
    np.testing.assert_array_equal(oracle.bin_matrix(X, optrs, ovals), b[:, None])


def test_signed_zeros_are_one_value(oracle):
    X = _col([-0.0, 0.0, 1.0, -1.0, -0.0])
    ptrs, vals, mins, _ = R.make_cuts(X, 256)
    assert_bitwise(vals, [0.0, 1.0, F32(1) + (F32(1) + R.EPS)])        # +0.0, never -0.0
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals)[:, 0], [1, 1, 2, 0, 1])
    _, ovals, _, _ = oracle.make_cuts(X, 256)
    assert np.all(ovals == vals)


def test_denormals(oracle):
    X = _col([3 * TINY, -TINY, 0.0, TINY, TINY])
    ptrs, vals, mins, _ = R.make_cuts(X, 256)
    end = F32(3 * TINY) + (F32(3 * TINY) + R.EPS)
    assert end == R.EPS and 3 * TINY > 0
    assert_bitwise(vals, [0.0, TINY, 3 * TINY, end])
    assert_bitwise(mins, [-TINY - (TINY + R.EPS)])
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals)[:, 0], [3, 0, 1, 2, 2])
    _, ovals, omins, _ = oracle.make_cuts(X, 256)
    assert np.all(ovals == vals) and np.all(omins == mins)


def test_flt_max(oracle):
    X = _col([0.0, FLT_MAX, -FLT_MAX])
    ptrs, vals, mins, _ = R.make_cuts(X, 256)
    assert_bitwise(vals, [0.0, FLT_MAX, np.inf])
    assert_bitwise(mins, [-np.inf])
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals)[:, 0], [1, 2, 0])
    _, ovals, omins, _ = oracle.make_cuts(X, 256)
    assert np.all(ovals == vals) and np.all(omins == mins)


def test_all_missing_constant_and_single_row(oracle):
    X = np.array([[np.nan, 3.0], [np.nan, 3.0], [np.nan, 3.0]], np.float32)
    ptrs, vals, mins, hm = R.make_cuts(X, 256)
    assert hm
    np.testing.assert_array_equal(ptrs, [0, 1, 2])
    assert_bitwise(vals, [R.EPS, F32(3) + (F32(3) + R.EPS)])
    assert_bitwise(mins, [-R.EPS, F32(3) - (F32(3) + R.EPS)])
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals), [[255, 0]] * 3)
    optrs, ovals, omins, _ = oracle.make_cuts(X, 256)
    np.testing.assert_array_equal(optrs, ptrs)
    assert np.all(ovals == vals) and np.all(omins == mins)
    one = np.array([[-2.5, 0.0, 7.0]], np.float32)
    ptrs, vals, mins, hm = R.make_cuts(one, 2)
    assert not hm
    assert_bitwise(vals, [F32(-2.5) + (F32(2.5) + R.EPS), R.EPS, F32(7) + (F32(7) + R.EPS)])
    np.testing.assert_array_equal(R.bin_matrix(one, ptrs, vals), [[0, 0, 0]])
    _, ovals, _, _ = oracle.make_cuts(one, 2)
    assert np.all(ovals == vals)


def test_missing_value_parameter():
    X = _col([1.0, -999.0, 2.0, 3.0, -999.0])
    ptrs, vals, mins, hm = R.make_cuts(X, 256, missing=-999.0)
    assert hm
    assert_bitwise(vals, [2.0, 3.0, F32(3) + (F32(3) + R.EPS)])
    np.testing.assert_array_equal(R.bin_matrix(X, ptrs, vals, missing=-999.0)[:, 0], [0, 255, 1, 2, 255])
    ptrs, vals, _, hm = R.make_cuts(_col([1.0, np.inf, 2.0]), 256, missing=np.inf)
    assert hm
    assert_bitwise(vals, [2.0, F32(2) + (F32(2) + R.EPS)])


def test_weighted_quantile_by_hand():
    """4 distinct values, weights 1, 2, 3, 2 (W = 8), nb = 2 (max_bin 2): the target 4 is first reached at value index 2
    (cumulative 1, 3, 6), so the one quantile cut is the next value; with weights 1, 3, 2, 2 it is reached exactly at index
    1 (cumulative 4 is not below 4), so the cut moves one value down"""
    X = _col([10, 20, 20, 30, 30, 30, 40, 40])
    ptrs, vals, _, _ = R.make_cuts(X, 2)
    assert_bitwise(vals, [40.0, F32(40) + (F32(40) + R.EPS)])
    w = np.array([1, 1.5, 1.5, 2 / 3, 2 / 3, 2 / 3, 1, 1], np.float32)
    w[5] = F32(2) - (w[3] + w[4])          # make each value's total exact: 1, 3, 2, 2
    assert float(np.float64(w[3]) + np.float64(w[4]) + np.float64(w[5])) == 2.0
    ptrs, vals, _, _ = R.make_cuts(X, 2, w)
    assert_bitwise(vals, [30.0, F32(40) + (F32(40) + R.EPS)])


def test_rank_summary_by_hand():
    d = np.arange(10, dtype=np.float32)
    v, w = R.rank_summary(d, np.ones(10, np.int64), 0, cap=4)
    # W = 10, targets 2.5, 5, 7.5, 10 over the cumulative 1..10 (the last value at the latest): indices 2, 4, 7, 9
    assert_bitwise(v, [0, 2, 4, 7, 9])
    np.testing.assert_array_equal(np.asarray(w, np.int64), [1, 2, 2, 3, 2])
    v, w = R.rank_summary(d, np.ones(10, np.int64), 0, cap=10)
    assert_bitwise(v, d)
    mv, mw = R.merge([(np.array([1, 3], np.float32), np.array([2, 5])), (np.array([0, 3, 4], np.float32), np.array([1, 1, 1]))])
    assert_bitwise(mv, [0, 1, 3, 4])
    np.testing.assert_array_equal(mw.astype(np.int64), [1, 2, 6, 1])


@pytest.mark.parametrize("weighted", [False, True])
def test_rank_recipe_is_exact_below_the_cap(weighted):
    """with no more than `cap` distinct values per shard and feature, the multi-rank cuts are the single-matrix cuts"""
    rng = np.random.default_rng(3)
    n = 4000
    X = (np.round(rng.standard_normal((n, 3)) * 6) / 6).astype(np.float32)
    X[rng.random((n, 3)) < 0.02] = np.nan
    X[5, 0], X[9, 1] = np.inf, -np.inf
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    bounds = [0, 1000, 1001, 2500, n]
    cap = max(len(np.unique(X[b:e, f][~np.isnan(X[b:e, f])])) for b, e in zip(bounds, bounds[1:]) for f in range(3))
    ptrs, vals, mins, _ = R.make_cuts(X, 16, w)
    rp, rv, rm = R.rank_cuts(X, 16, bounds, w, cap=cap)
    np.testing.assert_array_equal(rp, ptrs)
    assert_bitwise(rv, vals)
    assert_bitwise(rm, mins)
    rp, rv, rm = R.rank_cuts(X, 16, bounds, w, cap=cap // 3)        # capped: a different, still well-formed cut list
    assert np.all(np.diff(rv[rp[2]:rp[3]]) > 0)
