"""Constant-hessian growth on the dense g (run with `pytest -m gpu` on an H100).

For reg:squarederror without weights or row sampling every row has h == 1, so the round's gradients are written as a dense
float g and the gradient pass, the root histogram and the route scatter read 4 B per row instead of the (g,h) pair.  The
results must not change: every case is trained in a fresh process on that path and again with B200XGB_NO_CONSTH=1 (the (g,h)
path), and the exported trees and the cached margins must be identical bit for bit.  The cases cover feature layouts with
and without a tail, row counts that are not multiples of a 64-row root tile, routed (depth 6) and moved (depth 8, lossguide)
partitions, dart, a forest that shares the round's gradients, graph replay against direct launches, and a fresh root snapshot
after the training matrix is binned again."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3)
# name -> (rows, features, extra parameters, rounds); row counts are not multiples of 64 (the root tile) or 16
CASES = {}
for F, n in [(8, 37), (32, 1001), (36, 3001), (64, 4099), (100, 5003), (104, 4097), (130, 3003), (100, 300_001), (36, 1_100_003)]:
    CASES["depth6_F%d_n%d" % (F, n)] = (n, F, {}, 4)
for F, n in [(36, 6007), (100, 5003)]:
    CASES["depth8_F%d_n%d" % (F, n)] = (n, F, dict(max_depth=8), 3)
CASES["lossguide_F36"] = (6007, 36, dict(grow_policy="lossguide", max_depth=0, max_leaves=31), 3)
CASES["lossguide_F104"] = (4097, 104, dict(grow_policy="lossguide", max_depth=0, max_leaves=17), 3)
CASES["dart_F100"] = (3001, 100, dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7), 5)
CASES["forest_F36"] = (4099, 36, dict(num_parallel_tree=3, subsample=1.0, colsample_bynode=0.7, seed=5), 3)
CASES["missing_F100"] = (5003, 100, dict(missing_frac=0.1), 4)
CASES["rebin_F100"] = (5003, 100, dict(rebin_after=2), 4)

# Trains every listed case in this process and saves the models and cached margins.  argv: root, output .npz, case names
WORKER = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import sagemaker_xgboost_container_b200 as xgb
cases = json.loads(sys.argv[3])
be = xgb.get_backend()
out = {}
for name, (n, F, extra, rounds) in cases.items():
    extra = dict(extra)
    missing_frac = extra.pop("missing_frac", 0.0)
    rebin_after = extra.pop("rebin_after", None)
    rng = np.random.default_rng(n + F)
    X = (np.round(np.clip(rng.standard_normal((n, F)), -4, 4 - 1 / 32) * 32) / 32).astype(np.float32)
    y = (X @ (rng.standard_normal(F) / np.sqrt(F)) + 0.1 * rng.standard_normal(n)).astype(np.float32)
    if missing_frac:
        X[rng.random((n, F)) < missing_frac] = np.nan
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3)
    params.update(extra)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster(params, [d])
    for r in range(rounds):
        if r == rebin_after:          # the same matrix binned again (64 bins): the next tree takes a fresh root snapshot
            p, v, m, _ = be.dmatrix_get_cuts(d.handle, 64)
            be.dmatrix_set_cuts(d.handle, p, v, m)
        b.update(d, r)
    model = be.booster_export_model(b.handle)
    for k, a in model.items():
        out[name + "/" + k] = np.asarray(a)
    out[name + "/cache"] = be.booster_cached_margin(b.handle, d.handle, 1)
np.savez(sys.argv[2], **out)
"""


def _run(tmp_path, tag, cases, **env_extra):
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("B200XGB_NO_CONSTH", None)
    env.pop("B200XGB_NO_GRAPH", None)
    env.update(env_extra)
    out = str(tmp_path / (tag + ".npz"))
    r = subprocess.run([sys.executable, "-c", WORKER, ROOT, out, json.dumps(cases)], capture_output=True, text=True, timeout=1200, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return dict(np.load(out))


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _assert_same(a, b, what):
    assert sorted(a) == sorted(b)
    for k in sorted(a):
        np.testing.assert_array_equal(_bits(a[k]), _bits(b[k]), err_msg="%s: %s" % (what, k))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("dense_g")
    return {"dense": _run(tmp, "dense", CASES), "pairs": _run(tmp, "pairs", CASES, B200XGB_NO_CONSTH="1"),
            "direct": _run(tmp, "direct", {k: CASES[k] for k in ("depth6_F100_n5003", "depth8_F36_n6007", "lossguide_F36")},
                           B200XGB_NO_GRAPH="1")}


@pytest.mark.parametrize("case", sorted(CASES))
def test_dense_g_equals_pairs(runs, case):
    dense = {k: v for k, v in runs["dense"].items() if k.startswith(case + "/")}
    pairs = {k: v for k, v in runs["pairs"].items() if k.startswith(case + "/")}
    assert dense and (dense[case + "/left"] != -1).any(), "the case should grow splits"
    _assert_same(dense, pairs, case)


def test_graph_replay_equals_direct_launches(runs):
    direct = runs["direct"]
    names = {k.split("/")[0] for k in direct}
    assert len(names) == 3
    _assert_same({k: runs["dense"][k] for k in direct}, direct, "graph vs direct")


def test_rebinned_matrix_changes_the_trees(runs):
    """the 64-bin rounds really train on other bins (and still match the (g,h) path above)"""
    sb = runs["dense"]["rebin_F100/split_bin"]
    off = runs["dense"]["rebin_F100/tree_offset"]
    late = sb[off[2]:off[4]][runs["dense"]["rebin_F100/left"][off[2]:off[4]] != -1]
    assert late.size and late.max() < 64


def test_compute_gradient_still_returns_pairs(xgb):
    rng = np.random.default_rng(3)
    n, F = 1001, 8
    X = rng.standard_normal((n, F)).astype(np.float32)
    y = rng.standard_normal(n).astype(np.float32)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster(dict(BASE), [d])
    margin = rng.standard_normal(n).astype(np.float32)
    gp = xgb.get_backend().booster_compute_gradient(b.handle, d.handle, margin)
    assert gp.shape == (n, 1, 2)
    np.testing.assert_array_equal(gp[:, 0, 1], np.ones(n, np.float32))
    np.testing.assert_array_equal(gp[:, 0, 0], margin - y)


@pytest.mark.parametrize("n,F", [(1, 3), (37, 8), (1001, 100), (5003, 130), (300_001, 36)])
@pytest.mark.parametrize("mode", [2, 8, 10])
def test_g_only_root_histograms(xgb, oracle, n, F, mode):
    """XGB200BuildHistogramEx without row ids: mode 2 (hist_root_kernel<GONLY>) and 10 accumulate G alone from the dense g; mode
    8 runs hist_gather_kernel's contiguous G-only-payload pass, whose H plane adds rint(1.0f * sh) per row."""
    rng = np.random.default_rng(n + F)
    X = (np.round(np.clip(rng.standard_normal((n, F)), -4, 4 - 1 / 32) * 32) / 32).astype(np.float32)
    gpair = np.stack([rng.standard_normal(n).astype(np.float32) * 3, rng.random(n).astype(np.float32) + 0.01], axis=1)
    d = xgb.DMatrix(X, label=np.zeros(n, np.float32))
    b = xgb.Booster({"max_bin": 256}, [d])
    be = xgb.get_backend()
    hist, scales, _, kernel = be.build_histogram_ex(b.handle, d.handle, gpair, mode=mode)
    assert kernel == ("hist_gather_kernel" if mode == 8 else "hist_root_kernel<GONLY>")
    gq = np.rint(gpair[:, 0] * scales[0]).astype(np.int32)
    hq = np.full(n, np.rint(np.float32(1.0) * scales[1]), np.int32)
    ref = oracle.build_hist_fixed(be.dmatrix_get_bins(d.handle, 256), gq, hq)
    np.testing.assert_array_equal(hist[:, :, 0], ref[:, :, 0])
    if mode == 8:
        np.testing.assert_array_equal(hist[:, :, 1], ref[:, :, 1])
    else:
        assert not hist[:, :, 1].any()
