"""GPU tests of the quantile cuts and the binned matrix (csrc/quantile.cu, misc.cu bin / pad / transpose kernels) against
the exact restatement in tests/cuts_reference.py, bit for bit: cut values as uint32, ptrs, mins, has_missing and every bin
byte of all three binned copies the kernels read.

Covers continuous data on the quantile branch (millions of rows, duplicate runs across many sort tiles), weighted
quantiles whose targets fall exactly on cumulative boundaries, zero weights and new weights, +-inf with and without missing
values, +-0, denormals, the `missing` parameter, determinism across processes outside the exact regime, the multi-GPU cut
recipe run on one GPU (and on two, when there are two), and training on continuous weighted data against the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cuts_reference as R
from util import assert_same_structure, max_leaf_diff

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.asarray(a, np.float32).view(np.uint32)


def assert_cuts_equal(got, want):
    (p, v, m), (rp, rv, rm) = got[:3], want[:3]
    np.testing.assert_array_equal(p, rp)
    np.testing.assert_array_equal(_u32(v), _u32(rv))
    np.testing.assert_array_equal(_u32(m), _u32(rm))


def check(xgb, X, max_bin, w=None, missing=np.nan, d=None):
    """the device cuts and row-major bins of X (DMatrix d, or a new one) equal the restatement's"""
    if d is None:
        d = xgb.DMatrix(X, weight=w, missing=missing)
    got = _be().dmatrix_get_cuts(d.handle, max_bin)
    want = R.make_cuts(X, max_bin, w, missing)
    assert got[3] == want[3], "has_missing differs"
    assert_cuts_equal(got, want)
    bins = _be().dmatrix_get_bins(d.handle, max_bin)
    np.testing.assert_array_equal(bins, R.bin_matrix(X, want[0], want[1], missing))
    return d, want


# ------------------------------------------------------------------------------------------------ continuous data
N_BIG = 2_000_000


@pytest.fixture(scope="module")
def continuous():
    rng = np.random.default_rng(101)
    n = N_BIG
    X = np.empty((n, 4), np.float32)
    X[:, 0] = rng.standard_normal(n)                                         # nearly all distinct
    X[:, 1] = np.where(rng.random(n) < 0.6, 0.0, rng.standard_normal(n))      # 60 % zeros: one run across many sort tiles
    X[:, 1][rng.random(n) < 0.1] *= -0.0                                      # some of them -0.0
    X[:, 2] = rng.integers(0, 1_000_000, n).astype(np.float32) / 7            # about 860k distinct values
    X[:, 3] = np.round(rng.standard_normal(n) * 100) / 100                    # ~1000 long runs
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    assert R.in_exact_regime(w)
    return X, w


@pytest.mark.parametrize("max_bin", [2, 3, 16, 64, 255, 256, 1000])
@pytest.mark.parametrize("weighted", [False, True])
def test_continuous_quantile_branch(xgb, continuous, max_bin, weighted):
    X, w = continuous
    d, want = check(xgb, X, max_bin, w if weighted else None)
    assert np.diff(want[0]).max() == min(max_bin, 256)       # the quantile branch, every bin used
    if max_bin == 1000:                      # clamped to 256 bins, with a warning where the parameter comes in
        d.set_label(np.zeros(len(X), np.float32))
        with pytest.warns(UserWarning, match="max_bin=1000"):
            xgb.train({"max_bin": 1000, "max_depth": 2}, d, num_boost_round=1, verbose_eval=False)
        assert_cuts_equal(_be().dmatrix_get_cuts(d.handle, 256), want)


# ------------------------------------------------------------------------------------------------ weighted ties
def _tie_weights(L, seed):
    """L non-dyadic float32 weights whose float32 sum depends on the order it is taken in"""
    rng = np.random.default_rng(seed)
    ws = rng.uniform(0.1, 1.0, L).astype(np.float32)
    fwd, rev = F32(0), F32(0)
    for x in ws:
        fwd = F32(fwd + x)
    for x in ws[::-1]:
        rev = F32(rev + x)
    assert fwd != rev, "the weight list does not expose float summation"
    return ws


@pytest.mark.parametrize("nb,L", [(16, 3000), (256, 600)])
def test_weighted_ties_on_cumulative_boundaries(xgb, nb, L):
    """m = 2 nb distinct values, each with the same multiset of L weights shuffled over the rows: every target k W / nb is
    exactly the cumulative weight of the first 2k values, so a value total that is off by one rounding moves a cut"""
    ws = _tie_weights(L, nb)
    m = 2 * nb
    rng = np.random.default_rng(nb + 1)
    vals = np.repeat(np.arange(m, dtype=np.float32) * 0.25 - 7, L)
    w = np.tile(ws, m)
    perm = rng.permutation(len(vals))
    X, w = vals[perm][:, None].copy(), w[perm].copy()
    assert R.in_exact_regime(w)
    _, want = check(xgb, X, nb, w)
    # the exact answer: cut k is value 2k (the one after the value where the running weight lands on the target)
    np.testing.assert_array_equal(want[1][:-1], (np.arange(1, nb) * 2).astype(np.float32) * 0.25 - 7)


def test_zero_weights_and_new_weights(xgb):
    rng = np.random.default_rng(5)
    n = 300_000
    X = np.round(rng.standard_normal((n, 3)) * 50).astype(np.float32) / 50
    X[rng.random((n, 3)) < 0.01] = np.nan
    w = rng.uniform(0.25, 4.0, n).astype(np.float32)
    w[rng.random(n) < 0.3] = 0.0
    w[np.abs(X[:, 0]) > 2.5] = 0.0            # whole distinct values with zero weight
    d, first = check(xgb, X, 64, w)
    w2 = np.where(X[:, 1] > 0, w * 8, F32(0.125)).astype(np.float32)
    d.set_weight(w2)                          # the matrix is rebinned and the cuts follow the new weights
    _, second = check(xgb, X, 64, w2, d=d)
    assert not np.array_equal(first[1], second[1])


# ------------------------------------------------------------------------------------------------ special values
def _special_matrix(n, seed):
    rng = np.random.default_rng(seed)
    tiny = F32(2.0 ** -149)
    X = rng.standard_normal((n, 6)).astype(np.float32)
    X[rng.random(n) < 0.05, 0] = np.inf                                           # continuous + +inf (+ missing below)
    X[:, 1] = rng.integers(-3, 4, n).astype(np.float32)                            # list branch with +-inf
    X[rng.random(n) < 0.05, 1] = np.inf
    X[rng.random(n) < 0.05, 1] = -np.inf
    X[:, 2] = np.where(rng.random(n) < 0.5, F32(-0.0), F32(0.0))                  # signed zeros and a few ones
    X[rng.random(n) < 0.1, 2] = 1.0
    X[:, 3] = rng.integers(-40, 40, n).astype(np.float32) * tiny                  # denormals around zero
    X[:, 4] = np.where(rng.random(n) < 0.5, np.finfo(np.float32).max, -np.finfo(np.float32).max)
    X[:, 5] = rng.integers(0, 5, n).astype(np.float32)
    return X, rng


@pytest.mark.parametrize("max_bin", [16, 256])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("missing", ["nan", "none", -999.0, np.inf])
def test_special_values(xgb, max_bin, weighted, missing):
    X, rng = _special_matrix(200_000, 17)
    n = len(X)
    if missing == "none":
        miss = np.nan
    else:
        miss = np.nan if missing == "nan" else missing
        X[rng.random(n) < 0.03, 0] = miss                                        # +inf and missing values in one column
        X[rng.random(n) < 0.03, 1] = miss
        X[rng.random(n) < 0.5, 5] = miss
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    d, want = check(xgb, X, max_bin, w, missing=miss)
    assert want[3] == (missing != "none")
    ptrs, vals = want[0], want[1]
    if missing != np.inf:                     # +inf is a value with its own bin in the list branch, with or without missing values
        assert np.isposinf(vals[ptrs[2] - 2])
        b = _be().dmatrix_get_bins(d.handle, max_bin)[:, 1]
        pinf = np.isposinf(X[:, 1])
        assert len(np.unique(b[pinf])) == 1 and not np.any(b[np.isfinite(X[:, 1])] == b[pinf][0])


# ------------------------------------------------------------------------------------------------ every binned copy
@pytest.mark.parametrize("F", [1, 31, 32, 33, 36, 80, 96, 100, 101, 104, 130])
def test_every_binned_copy(xgb, F):
    rng = np.random.default_rng(F)
    base = rng.standard_normal((4000, F)).astype(np.float32)
    base[rng.random(base.shape) < 0.02] = np.nan
    ptrs, vals, mins, _ = R.make_cuts(base, 16)
    # probe rows: every cut, and the floats just below and just above it, in every feature
    k = int(np.diff(ptrs).max())
    probe = np.full((3 * k, F), np.nan, np.float32)
    for f in range(F):
        c = vals[ptrs[f]:ptrs[f + 1]]
        col = np.concatenate([c, np.nextafter(c, F32(-np.inf)), np.nextafter(c, F32(np.inf))])
        probe[:len(col), f] = col
    X = np.concatenate([base, probe, base[:777]])
    d = xgb.DMatrix(X)
    _be().dmatrix_set_cuts(d.handle, ptrs, vals, mins)
    want = R.bin_matrix(X, ptrs, vals)
    n = len(X)
    np.testing.assert_array_equal(_be().dmatrix_get_bins(d.handle, 16), want)          # row-major main block + tail
    aligned, col = _be().dmatrix_get_bin_copies(d.handle, 16)
    np.testing.assert_array_equal(col, want.T)                                            # column-major copy
    if 73 <= F <= 104:                       # 96 B main block: the 128 B line-aligned copy
        assert aligned is not None and aligned.shape == (n, 128)
        main = min(F, 96)
        np.testing.assert_array_equal(aligned[:, :main], want[:, :main])
        if F >= 101:                         # an 8-wide tail sits at offset 96, its unused slots zero
            np.testing.assert_array_equal(aligned[:, 96:F], want[:, 96:F])
            assert not aligned[:, F:].any()
        else:                                # pad slots of the main block and the rest of the line are zero; a 4-wide tail is not there
            assert not aligned[:, main:].any()
    else:
        assert aligned is None


# ------------------------------------------------------------------------------------------------ determinism
DET_SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import sagemaker_xgboost_container_b200 as xgb
rng = np.random.default_rng(404)
n = 3_000_000
X = np.round(rng.standard_normal((n, 3)) * 300).astype(np.float32) / 300
X[:, 2] = rng.standard_normal(n)
w = np.ldexp(rng.uniform(1, 2, n), rng.integers(-20, 21, n)).astype(np.float32)
d = xgb.DMatrix(X, weight=w)
p, v, m, hm = xgb.get_backend().dmatrix_get_cuts(d.handle, 256)
np.savez(sys.argv[2], p=p, v=v, m=m, inexact=np.array(not __import__("cuts_reference").in_exact_regime(w)))
"""


def test_weighted_cuts_identical_across_processes(tmp_path):
    """outside the exact regime (weights 2^-20 .. 2^21 on 3M rows) the double sums round, but the same way every time"""
    outs = []
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    for i in range(2):
        out = str(tmp_path / ("cuts%d.npz" % i))
        r = subprocess.run([sys.executable, "-c", DET_SCRIPT, ROOT, out], capture_output=True, text=True, timeout=600, env=env)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        outs.append(np.load(out))
    assert bool(outs[0]["inexact"])
    np.testing.assert_array_equal(outs[0]["p"], outs[1]["p"])
    np.testing.assert_array_equal(_u32(outs[0]["v"]), _u32(outs[1]["v"]))
    np.testing.assert_array_equal(_u32(outs[0]["m"]), _u32(outs[1]["m"]))


# ------------------------------------------------------------------------------------------------ multi-rank recipe
def _rank_data(n, F, levels, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, F)).astype(np.float32)
    if levels:
        X = (np.round(X * levels / 8) / (levels / 8)).astype(np.float32)
    X[rng.random((n, F)) < 0.02] = np.nan
    X[rng.random((n, F)) < 0.01] = np.inf
    X[rng.random((n, F)) < 0.01] = -np.inf
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    return X, w


@pytest.mark.parametrize("max_bin", [16, 256])
@pytest.mark.parametrize("weighted", [False, True])
def test_rank_recipe_matches_restatement(xgb, max_bin, weighted):
    """shards with far more than 2048 distinct values: the capped summaries, their merge and the cuts, bit for bit"""
    X, w = _rank_data(60_000, 5, 0, 31)
    w = w if weighted else None
    bounds = [0, 9000, 9001, 30000, 30000, 60000]
    d = xgb.DMatrix(X, weight=w)
    got = _be().dmatrix_rank_cuts(d.handle, max_bin, bounds)
    assert_cuts_equal(got, R.rank_cuts(X, max_bin, bounds, w))


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("nranks", [2, 3, 8])
def test_rank_recipe_equals_single_gpu_below_the_cap(xgb, weighted, nranks):
    """at most 2048 distinct values per shard and feature: N-rank cuts are the 1-GPU cuts bit for bit"""
    X, w = _rank_data(200_000, 4, 1500, 37)
    w = w if weighted else None
    d = xgb.DMatrix(X, weight=w)
    bounds = [len(X) * r // nranks for r in range(nranks + 1)]
    single = _be().dmatrix_get_cuts(d.handle, 256)
    assert_cuts_equal(_be().dmatrix_rank_cuts(d.handle, 256, bounds), single)
    assert_cuts_equal(single, R.make_cuts(X, 256, w))


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_rank_cuts_equal_one_gpu_simulation(xgb, tmp_path):
    """real two-rank cuts on continuous weighted data (over the summary cap) equal the one-GPU run of the same recipe"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "cuts.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29623", os.path.join(ROOT, "tests", "helpers", "cuts_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    got = np.load(out)
    X, w = _rank_data(60_000, 5, 0, 31)
    d = xgb.DMatrix(X, weight=w)
    want = _be().dmatrix_rank_cuts(d.handle, 256, [0, 30000, 60000])
    assert_cuts_equal((got["p"], got["v"], got["m"]), want)


# ------------------------------------------------------------------------------------------------ training
def test_training_on_continuous_weighted_data(xgb, oracle):
    rng = np.random.default_rng(77)
    n, F = 60_000, 8
    X = rng.standard_normal((n, F)).astype(np.float32)
    X[:, 0] = np.round(X[:, 0] * 3) / 3                        # long duplicate runs
    X[rng.random(n) < 0.5, 1] = 0.0
    X[rng.random((n, F)) < 0.01] = np.nan
    y = (X[:, 2] - 0.5 * np.nan_to_num(X[:, 0]) + np.where(np.isnan(X[:, 1]), 1.0, np.nan_to_num(X[:, 1])) ** 2
         + 0.1 * rng.standard_normal(n)).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    params = dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=64)
    d = xgb.DMatrix(X, label=y, weight=w)
    bst = xgb.train(params, d, num_boost_round=5, verbose_eval=False)
    cuts = R.make_cuts(X, 64, w)
    assert_cuts_equal(_be().dmatrix_get_cuts(d.handle, 64), cuts)
    ref = oracle.train(params, X, y, 5, weights=w).model()
    m = _be().booster_export_model(bst.handle)
    assert_same_structure(m, ref)
    assert max_leaf_diff(m, ref) <= 1e-5
