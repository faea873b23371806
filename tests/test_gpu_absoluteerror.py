"""reg:absoluteerror on the GPU (run with `pytest -m gpu` on an H100): the select kernels through XGB200SegmentedQuantile and
whole models against tests/absoluteerror_reference.py bit for bit, the base score, the constant-hessian and (g,h) paths, graph
replay, checkpoint resume, model IO, SHAP, the mae metric, the container's string hyperparameters, and two ranks."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import absoluteerror_reference as A
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_bits(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return a.shape == b.shape and bool(np.all((_u32(a) == _u32(b)) | (np.isnan(a) & np.isnan(b))))


def _data(n, F, seed, missing_frac=0.0):
    X, y = synth(n, F, seed, "reg", missing_frac=missing_frac)
    y = (y + np.random.default_rng(seed).laplace(0, 0.5, n)).astype(f32)
    return X, y


# ---------------------------------------------------------------------------------------------------------------- the select
def _select_sets():
    rng = np.random.default_rng(11)
    yield "one", np.array([2.5], f32), None, 1
    yield "two", np.array([1.0, -3.0], f32), None, 1
    yield "equal", np.full(1000, 0.75, f32), None, 1
    yield "signed_zeros", np.array([0.0, -0.0] * 500 + [1.0], f32), None, 1
    yield "extremes", np.array([3e38, -3e38, 1e-45, -1e-45, 0.0, np.inf, -np.inf], f32), None, 1
    v = np.round(rng.standard_normal(200_000), 1).astype(f32)                 # ties in every segment
    yield "ties_64", v, rng.integers(-1, 64, len(v)), 64
    v = rng.standard_normal(300_000).astype(f32)
    yield "segs_65536_with_empty", v, rng.integers(0, 65536 - 100, len(v)), 65536
    v = rng.standard_normal(1_500_000).astype(f32)                           # above 2^20: the 18-bit grid
    yield "big_1000", v, rng.integers(0, 1000, len(v)), 1000


@pytest.mark.parametrize("weighted", [False, True])
def test_segmented_quantile_bit_exact(xgb, weighted):
    rng = np.random.default_rng(12)
    for name, v, seg, S in _select_sets():
        w = None
        if weighted:
            w = rng.uniform(0.0, 3.0, len(v)).astype(f32)
            w[rng.random(len(v)) < 0.05] = 0.0                                 # left out
        got = _be().segmented_quantile(v, seg, w, S, 0.5)
        want = A.segmented_quantile(v, seg, w, S, 0.5)
        assert _same_bits(got, want), (name, np.nonzero(~((_u32(got) == _u32(want)) | (np.isnan(got) & np.isnan(want))))[0][:5])


@pytest.mark.parametrize("alpha", [0.0, 0.1, 0.9, 1.0])
def test_segmented_quantile_other_alpha(xgb, alpha):
    rng = np.random.default_rng(13)
    v = rng.standard_normal(50_000).astype(f32)
    seg = rng.integers(0, 7, len(v))
    a32 = float(f32(alpha))                   # the entry point takes alpha as a float
    assert _same_bits(_be().segmented_quantile(v, seg, None, 9, alpha), A.segmented_quantile(v, seg, None, 9, a32))


# ---------------------------------------------------------------------------------------------------------------- whole models
BASE = dict(objective="reg:absoluteerror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3)
MODEL_CASES = {
    "depth6": (20000, 8, {}, {}),
    "depth8": (20000, 8, dict(max_depth=8), {}),
    "lossguide": (20000, 8, dict(grow_policy="lossguide", max_depth=0, max_leaves=40), {}),
    "missing": (20000, 8, {}, dict(missing_frac=0.15)),
    "weights": (20000, 8, {}, dict(weighted=True)),
    "weights_lossguide": (20000, 8, dict(grow_policy="lossguide", max_depth=0, max_leaves=24), dict(weighted=True)),
    "subsample_mcw0": (3000, 8, dict(subsample=0.5, min_child_weight=0, max_depth=8, seed=3), {}),
    "base_margin": (20000, 8, {}, dict(base_margin=True)),
    "rows_above_2p20": (1_100_003, 8, dict(max_depth=6), {}),
    # forests: three trees per round, each on its own row sample, leaves and refresh at fl(eta / 3)
    "forest_sampled": (20000, 8, dict(num_parallel_tree=3, subsample=0.6, seed=5), {}),
    "forest_weights": (20000, 8, dict(num_parallel_tree=3, subsample=0.7, seed=6), dict(weighted=True)),
    "forest_unsampled": (20000, 8, dict(num_parallel_tree=2, seed=5), {}),
    # dart: residuals at the margin without the dropped trees, refreshed leaves entering the margin at the new-tree weight
    "dart": (20000, 8, dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7), {}),
    "dart_weighted_forest_norm": (20000, 8, dict(booster="dart", rate_drop=0.4, sample_type="weighted", normalize_type="forest", seed=8),
                                  dict(weighted=True)),
}


@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_model_matches_reference(xgb, case):
    n, F, extra, opts = MODEL_CASES[case]
    X, y = _data(n, F, 21, opts.get("missing_frac", 0.0))
    rng = np.random.default_rng(22)
    w = rng.integers(1, 5, n).astype(f32) if opts.get("weighted") else None
    bm = rng.normal(0, 1, n).astype(f32) if opts.get("base_margin") else None
    params = dict(BASE, **extra)
    d = xgb.DMatrix(X, label=y, weight=w, base_margin=bm)
    bst = xgb.Booster(params, [d])
    ref = A.AbsErrorTrainer(params, X, y, weight=w, base_margin=bm, bins=_be().dmatrix_get_bins(d.handle, 256),
                            cuts=_be().dmatrix_get_cuts(d.handle, 256))
    rounds = 2 if n > 1_000_000 else 5 if extra.get("booster") == "dart" else 4
    for r in range(rounds):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert m["base_score"] == mr["base_score"]
    assert_same_structure(m, mr)
    empty = 0
    for tid, vals in ref.leaves.items():
        off = int(mr["tree_offset"][tid])
        leaves = np.nonzero(mr["left"][off:int(mr["tree_offset"][tid + 1])] == -1)[0]
        empty += len(leaves) - len(vals)
        for nid, v in vals.items():
            assert _u32(m["split_cond"][off + nid]) == _u32(v), (tid, nid)
    # a leaf without sampled rows keeps its Newton value, which the oracle reaches only to 1e-5 (fixed-point vs double sums)
    assert max_leaf_diff(m, mr) <= 1e-5
    cache = _be().booster_cached_margin(bst.handle, d.handle, 1)[:, 0]
    if empty == 0:
        assert _same_bits(cache, ref.m)
    else:          # unsampled rows in a leaf without sampled rows take its Newton value: equal to 1e-5 per tree
        assert "subsample" in extra
        np.testing.assert_allclose(cache, ref.m, rtol=0, atol=1e-5 * len(ref.weights))
    assert _same_bits(_be().booster_tree_weights(bst.handle), ref.weights)
    pred = bst.predict(d, output_margin=True).reshape(-1)
    if extra.get("booster") == "dart":       # predict sums fl(w_t * leaf_t) afresh; the cache carries each round's weight changes
        import dart_reference as DR
        assert _same_bits(pred, DR.predict_margin(m, X, _be().booster_tree_weights(bst.handle), base_margin=bm)[:, 0])
    else:
        assert _same_bits(pred, cache)


@pytest.mark.parametrize("weighted", [False, True])
def test_base_score_is_median(xgb, weighted):
    X, y = _data(30001, 4, 31)
    w = np.random.default_rng(32).uniform(0, 4, len(y)).astype(f32) if weighted else None
    bst = xgb.train(dict(BASE), xgb.DMatrix(X, label=y, weight=w), num_boost_round=1, verbose_eval=False)
    assert f32(_be().booster_export_model(bst.handle)["base_score"]) == A.base_score(y, w)


def test_nan_label_rejected(xgb):
    X, y = _data(100, 3, 33)
    y[7] = np.nan
    with pytest.raises(xgb.core.XGBoostError, match="must not be NaN"):
        xgb.train(dict(BASE), xgb.DMatrix(X, label=y), num_boost_round=1, verbose_eval=False)


# ---------------------------------------------------------------------------------------------------------------- paths in fresh processes
PATH_CASES = {
    "depth6": (30001, 36, {}, 4),
    "depth8": (20011, 100, dict(max_depth=8), 3),
    "lossguide": (20011, 36, dict(grow_policy="lossguide", max_depth=0, max_leaves=31), 3),
    "dart": (20011, 100, dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7), 5),
    "forest": (20011, 36, dict(num_parallel_tree=3, colsample_bynode=0.7, seed=5), 3),
    "forest_sampled": (20011, 36, dict(num_parallel_tree=3, subsample=0.6, seed=5), 3),
    "missing": (20011, 36, dict(missing_frac=0.1), 4),
}
WORKER = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import sagemaker_xgboost_container_b200 as xgb
from test_gpu_absoluteerror import _data, BASE
be = xgb.get_backend()
out = {}
for name, (n, F, extra, rounds) in json.loads(sys.argv[3]).items():
    extra = dict(extra); mf = extra.pop("missing_frac", 0.0)
    X, y = _data(n, F, n + F, mf)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster(dict(BASE, **extra), [d])
    for r in range(rounds):
        b.update(d, r)
    m = be.booster_export_model(b.handle)
    for k in ("left", "split_index", "split_cond", "base_weight"):
        out[name + "/" + k] = m[k]
    out[name + "/margin"] = be.booster_cached_margin(b.handle, d.handle, 1)
np.savez(sys.argv[2], **out)
"""


def _run_worker(tmp_path, tag, env_extra):
    env = dict(os.environ)
    env.pop("B200XGB_NO_CONSTH", None); env.pop("B200XGB_NO_GRAPH", None)
    env.update(env_extra)
    out = str(tmp_path / (tag + ".npz"))
    r = subprocess.run([sys.executable, "-c", WORKER, ROOT, out, json.dumps(PATH_CASES)], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return dict(np.load(out))


def test_constant_hessian_graph_and_direct_paths_agree(xgb, tmp_path):
    base = _run_worker(tmp_path, "default", {})
    for tag, env in (("gh", {"B200XGB_NO_CONSTH": "1"}), ("direct", {"B200XGB_NO_GRAPH": "1"})):
        other = _run_worker(tmp_path, tag, env)
        for k in base:
            assert _same_bits(base[k], other[k]) if base[k].dtype == np.float32 else np.array_equal(base[k], other[k]), (tag, k)


# ---------------------------------------------------------------------------------------------------------------- resume, IO, SHAP, metric
def test_resume_equals_uninterrupted(xgb, tmp_path):
    X, y = _data(20000, 8, 41)
    d = xgb.DMatrix(X, label=y)
    full = xgb.train(dict(BASE), d, num_boost_round=6, verbose_eval=False)
    half = xgb.train(dict(BASE), d, num_boost_round=3, verbose_eval=False)
    path = str(tmp_path / "half.json")
    half.save_model(path)
    resumed = xgb.train(dict(BASE), d, num_boost_round=3, xgb_model=path, verbose_eval=False)
    a, b = _be().booster_export_model(full.handle), _be().booster_export_model(resumed.handle)
    assert_same_structure(b, a)
    assert _same_bits(a["split_cond"], b["split_cond"])


def test_model_io_round_trips(xgb, tmp_path):
    X, y = _data(5000, 6, 42)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=4, verbose_eval=False)
    p0 = bst.predict(d)
    for fmt in ("json", "ubj"):
        path = str(tmp_path / ("m." + fmt))
        bst.save_model(path)
        assert _same_bits(xgb.Booster(model_file=path).predict(d), p0)
    assert _same_bits(pickle.loads(pickle.dumps(bst)).predict(d), p0)
    doc = json.loads(open(str(tmp_path / "m.json")).read())
    assert doc["learner"]["objective"] == {"name": "reg:absoluteerror"}
    # an upstream-style document: a squared-error model whose objective block is replaced by reg:absoluteerror's
    sq = xgb.train(dict(BASE, objective="reg:squarederror", max_depth=3), d, num_boost_round=2, verbose_eval=False)
    path = str(tmp_path / "sq.json")
    sq.save_model(path)
    doc = json.loads(open(path).read())
    doc["learner"]["objective"] = {"name": "reg:absoluteerror"}
    doc["version"] = [3, 0, 5]
    with open(path, "w") as f:
        json.dump(doc, f)
    loaded = xgb.Booster(model_file=path)
    assert _same_bits(loaded.predict(d), sq.predict(d))
    assert json.loads(loaded.save_config())["learner"]["objective"]["name"] == "reg:absoluteerror"


def test_shap_and_metric(xgb, oracle):
    X, y = _data(400, 6, 43)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(BASE, max_depth=4), d, num_boost_round=3, verbose_eval=False)
    contrib = bst.predict(d, pred_contribs=True)
    margin = bst.predict(d, output_margin=True)
    np.testing.assert_allclose(contrib.sum(axis=1), margin, rtol=0, atol=1e-5)
    m = _be().booster_export_model(bst.handle)
    bf = oracle.shap_bruteforce(m, X[:50])[:, 0, :]
    np.testing.assert_allclose(contrib[:50], bf, rtol=0, atol=1e-5)
    line = bst.eval(d, "train")
    assert "train-mae:" in line
    got = float(line.split("train-mae:")[1].split()[0])
    assert abs(got - float(np.mean(np.abs(y.astype(np.float64) - margin.astype(np.float64))))) <= 1e-6 * max(1.0, got)


def test_sklearn_and_string_hyperparameters(xgb):
    X, y = _data(5000, 6, 44)
    from sagemaker_xgboost_container_b200 import sklearn as skl
    reg = skl.XGBRegressor(objective="reg:absoluteerror", n_estimators=3, max_depth=4)
    reg.fit(X, y)
    assert reg.predict(X).shape == (5000,)
    params = {"objective": "reg:absoluteerror", "max_depth": "4", "eta": "0.3", "subsample": "0.8", "eval_metric": "mae"}
    bst = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    assert np.all(np.isfinite(bst.predict(xgb.DMatrix(X))))


# ---------------------------------------------------------------------------------------------------------------- two ranks
# No row sampling: each rank draws its rows at index r + (rank << 40), so a sample differs between 1 and 2 GPUs.  Rows of
# weight 0 are left out of the refresh as unsampled rows are.
TWO_RANK_PARAMS = dict(BASE, max_depth=5, seed=3)


def two_rank_data():
    """Shards that keep the per-rank cut summary exact: at most 2048 distinct values per feature (DESIGN.md §5); weights with
    zeros, so the h_q rule, the weighted base score and the left-out rows all cross ranks."""
    X, y = _data(40000, 10, 45)
    rng = np.random.default_rng(46)
    w = rng.integers(1, 4, len(y)).astype(f32)
    w[rng.random(len(y)) < 0.1] = 0.0
    return X, y, w


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks(xgb, tmp_path):
    """Two ranks train the 1-GPU model bit for bit: the select's histograms are all-reduced in int64."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29619", os.path.join(ROOT, "tests", "helpers", "absoluteerror_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y, w = two_rank_data()
    single = xgb.train(TWO_RANK_PARAMS, xgb.DMatrix(X, label=y, weight=w), num_boost_round=3, verbose_eval=False)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(xgb.Booster(model_file=out).handle)
    assert m1["base_score"] == m2["base_score"]
    assert_same_structure(m2, m1)
    assert _same_bits(m2["split_cond"], m1["split_cond"])
