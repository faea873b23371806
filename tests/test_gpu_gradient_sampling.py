"""sampling_method=gradient_based on the GPU (run with `pytest -m gpu` on an H100): the select and sampling kernels through
XGB200GradientBasedSample and the training path's tree-0 sample through XGB200BoosterComputeGradient, bit for bit against
tests/gradient_sampling_reference.py; whole models against the restatement's trainer; the sample's statistics; accuracy at
subsample 0.1; determinism across retraining, graph replay and resume; no change at subsample 1; the Python surface."""
import json
import os
import pickle
import subprocess
import sys
import warnings

import numpy as np
import pytest

import gradient_sampling_reference as G
from forest_reference import FOREST_ROW_STREAM
from split_reference import grad_bits_for, scales_for
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


# ---------------------------------------------------------------------------------------------------------------- the kernels
def _pair_sets(xgb):
    rng = np.random.default_rng(1)
    n = 1_000_000
    yield "random_1m", np.stack([rng.standard_normal(n), rng.uniform(0, 2, n)], 1), 0.3
    yield "random_1m_sub0.01", np.stack([rng.standard_normal(n), rng.uniform(0, 2, n)], 1), 0.01
    n = 1_500_001                                                  # above 2^20 rows: the 18-bit grid
    yield "random_1.5m_wide", np.stack([rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n)), rng.uniform(0, 2, n)], 1), 0.2
    X, y = synth(200_000, 10, 2, "bin")
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster(dict(objective="binary:logistic"), [d])
    m = rng.normal(0, 2, len(y)).astype(f32)
    yield "logistic", _be().booster_compute_gradient(b.handle, d.handle, m)[:, 0], 0.3
    X, y = synth(100_000, 10, 3, "multi", K=3)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster(dict(objective="multi:softprob", num_class=3), [d])
    gp = _be().booster_compute_gradient(b.handle, d.handle, rng.normal(0, 1, (len(y), 3)).astype(f32))
    for c in range(3):
        yield "softprob_class%d" % c, gp[:, c], 0.3
    yield "zeros", np.zeros((1000, 2)), 0.3
    z = np.stack([rng.standard_normal(5000), rng.uniform(0, 1, 5000)], 1)
    z[rng.random(5000) < 0.5] = 0
    yield "half_zero_pairs", z, 0.2
    yield "k0", np.stack([rng.standard_normal(50), np.ones(50)], 1), 0.01
    yield "k_ge_n", np.stack([rng.standard_normal(1000), np.ones(1000)], 1), 0.9999
    yield "k_ge_nonzero", np.concatenate([np.stack([rng.standard_normal(100), np.ones(100)], 1), np.zeros((900, 2))]), 0.5
    yield "ties", np.tile([[0.5, 1.0]], (10000, 1)), 0.25
    yield "ties_rounded", np.stack([np.round(rng.standard_normal(100000), 1), np.ones(100000)], 1), 0.3
    nf = np.stack([rng.standard_normal(3000), rng.uniform(0, 1, 3000)], 1)
    nf[:5, 0], nf[5:8, 0], nf[8:10, 1] = np.inf, np.nan, np.inf
    yield "non_finite", nf, 0.3
    yield "all_non_finite", np.full((10, 2), np.inf), 0.3
    de = np.zeros((4000, 2))
    de[:, 0] = np.arange(1, 4001, dtype=np.uint32).view(np.float32)
    de[2000:, 1] = 2e-19
    de[3000:, 0] = 1e-30
    yield "denormal", de, 0.1
    yield "one_huge", np.concatenate([np.stack([np.full(999, 1e-3), np.ones(999)], 1), [[3e38, 1.0]]]), 0.1


def test_kernels_bit_exact(xgb):
    for name, gp, sub in _pair_sets(xgb):
        gp = np.ascontiguousarray(gp, f32)
        for seed, stream in ((0, 0x2000), (7, FOREST_ROW_STREAM + 3)) if name == "random_1m" else ((3, 0x2005),):
            u, out = _be().gradient_based_sample(gp, sub, seed, stream)
            ru, rout = G.gradient_based_sample(gp, sub, seed, stream)
            assert _u32(u) == _u32(ru), (name, float(u), float(ru))
            bad = np.nonzero(~np.all((_u32(out) == _u32(rout)) | (np.isnan(out) & np.isnan(rout)), axis=1))[0]
            assert len(bad) == 0, (name, bad[:5], out[bad[:5]], rout[bad[:5]])


def test_statistics_on_one_seed(xgb):
    rng = np.random.default_rng(5)
    n = 1_000_000
    gp = np.stack([rng.standard_normal(n), rng.uniform(0.01, 2.0, n)], 1).astype(f32)
    u, out = _be().gradient_based_sample(gp, 0.2, 11, 0x2000)
    r = G.rag(gp).astype(np.float64)
    p = np.minimum(1.0, r / float(u))
    kept = out[:, 1] != 0
    k = G.target(n, 0.2)
    assert abs(int(kept.sum()) - k) <= 5 * np.sqrt(np.sum(p * (1 - p)))
    g = gp[:, 0].astype(np.float64)
    assert abs(out[:, 0].astype(np.float64).sum() - g.sum()) <= 5 * np.sqrt(np.sum(g * g * (1 - p) / p))
    above = r >= float(u)
    assert above.any() and np.array_equal(_u32(out[above]), _u32(gp[above]))


@pytest.mark.parametrize("objective,K", [("binary:logistic", 1), ("multi:softprob", 3), ("reg:absoluteerror", 1)])
def test_training_path_tree0_sample_bit_exact(xgb, objective, K):
    X, y = synth(30011, 6, 4, "multi" if K > 1 else "bin", K=max(K, 2))
    d = xgb.DMatrix(X, label=y)
    p = dict(objective=objective, seed=13, subsample=0.3)
    if K > 1:
        p["num_class"] = K
    sampled = xgb.Booster(dict(p, sampling_method="gradient_based"), [d])
    plain = xgb.Booster(dict(p, subsample=1.0), [d])
    m = np.random.default_rng(6).normal(0, 1, (len(y), K)).astype(f32)
    for rnd in (0, 4):
        full = _be().booster_compute_gradient(plain.handle, d.handle, m, rnd)
        got = _be().booster_compute_gradient(sampled.handle, d.handle, m, rnd)
        want = G.sample_classes(full, 0.3, 13, 0x2000 + rnd)
        assert _same_bits(got, want), (objective, rnd)


# ---------------------------------------------------------------------------------------------------------------- whole models
BASE = dict(tree_method="hist", max_bin=256, max_depth=6, eta=0.3, subsample=0.3, sampling_method="gradient_based", seed=17)


def _aft(n, F, seed):
    X, y = synth(n, F, seed, "reg")
    rng = np.random.default_rng(seed)
    t = np.exp(1.0 + 0.5 * y + 0.3 * rng.standard_normal(n)).astype(f32)
    lo, hi = t.copy(), t.copy()
    c = rng.random(n)
    hi[c < 0.3] = np.inf
    lo[(c >= 0.3) & (c < 0.4)] = 0
    iv = (c >= 0.4) & (c < 0.5)
    hi[iv] = t[iv] * 1.5
    return X, lo, hi


MODEL_CASES = {
    "squarederror": dict(objective="reg:squarederror", base_score=0.5),
    "logistic": dict(objective="binary:logistic", base_score=0.5),
    "lossguide": dict(objective="binary:logistic", base_score=0.5, grow_policy="lossguide", max_depth=0, max_leaves=24),
    "forest3": dict(objective="reg:squarederror", base_score=0.5, num_parallel_tree=3),
    "dart": dict(objective="binary:logistic", base_score=0.5, booster="dart", rate_drop=0.4, one_drop=1),
    "aft": dict(objective="survival:aft", base_score=1.0, max_depth=4),
    "constraints_colsample": dict(objective="reg:squarederror", base_score=0.5, colsample_bytree=0.8, monotone_constraints="(1,0,-1,0,0,0,0,0)",
                                  interaction_constraints="[[0,1,2],[3,4,5,6,7]]"),
}


@pytest.mark.parametrize("case", list(MODEL_CASES))
def test_model_matches_reference(xgb, case):
    params = dict(BASE, **MODEL_CASES[case])
    n, F = 20000, 8
    if params["objective"] == "survival:aft":
        X, lo, hi = _aft(n, F, 31)
        d = xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
        m0 = np.log(f32(1.0))
    else:
        X, y = synth(n, F, 31, "bin" if "logistic" in params["objective"] else "reg")
        d = xgb.DMatrix(X, label=y)
        m0 = f32(0) if "logistic" in params["objective"] else f32(0.5)
    helper = xgb.Booster(dict(params, subsample=1.0, sampling_method="uniform"), [d])

    def grad(m, rnd):
        return _be().booster_compute_gradient(helper.handle, d.handle, m.reshape(-1, 1), rnd)[:, 0]

    bst = xgb.Booster(params, [d])
    ref = G.GbsTrainer(params, X, grad, m0, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256))
    for r in range(3):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= 1e-5
    cache = _be().booster_cached_margin(bst.handle, d.handle, 1)[:, 0]
    if ref.exact and params.get("booster") != "dart":
        assert _same_bits(m["split_cond"], mr["split_cond"]) and _same_bits(cache, ref.m)
    np.testing.assert_allclose(cache, ref.m, rtol=0, atol=2e-5)


@pytest.mark.parametrize("weighted,P", [(False, 1), (True, 1), (True, 3)])
def test_absoluteerror_matches_reference(xgb, weighted, P):
    import absoluteerror_reference as A
    X, y = synth(20000, 8, 41, "reg")
    y = (y + np.random.default_rng(41).laplace(0, 0.5, len(y))).astype(f32)
    w = np.random.default_rng(42).integers(1, 6, len(y)).astype(f32) if weighted else None
    params = dict(BASE, objective="reg:absoluteerror", num_parallel_tree=P)
    d = xgb.DMatrix(X, label=y, weight=w)
    bst = xgb.Booster(params, [d])
    ref = G.GbsAbsErrorTrainer(params, X, y, weight=w, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256))
    for r in range(3):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert m["base_score"] == mr["base_score"]
    assert_same_structure(m, mr)
    for tid, vals in ref.leaves.items():
        off = int(mr["tree_offset"][tid])
        for nid, v in vals.items():
            assert _u32(m["split_cond"][off + nid]) == _u32(v), (tid, nid)
    assert max_leaf_diff(m, mr) <= 1e-5
    np.testing.assert_allclose(_be().booster_cached_margin(bst.handle, d.handle, 1)[:, 0], ref.m, rtol=0, atol=2e-5)
    if weighted:           # the refresh weighs by the instance weight: weighing by h = w / p would give other leaves
        differs = 0
        for tid, leaf, gp, resid in ref.samples:
            sh = scales_for(np.max(np.abs(gp[:, 0])), np.max(gp[:, 1]), grad_bits_for(len(gp)))[1]
            by_h = A.refresh(leaf, resid, gp[:, 1], True, sh)
            differs += sum(_u32(f32(q * ref.lr)) != _u32(ref.leaves[tid][nid]) for nid, q in by_h.items())
        assert differs > 0


# ---------------------------------------------------------------------------------------------------------------- determinism and no change
def _train(xgb, params, d, rounds, **kw):
    return xgb.train(params, d, num_boost_round=rounds, verbose_eval=False, **kw)


def _bytes(bst):
    return bytes(bst.save_raw("ubj"))


def test_retrain_and_resume_give_identical_models(xgb, tmp_path):
    X, y = synth(50000, 12, 51, "bin")
    d = xgb.DMatrix(X, label=y)
    params = dict(BASE, objective="binary:logistic")
    a, b = _train(xgb, params, d, 6), _train(xgb, params, d, 6)
    assert _bytes(a) == _bytes(b)
    half = _train(xgb, params, d, 3)
    path = str(tmp_path / "half.json")
    half.save_model(path)
    resumed = _train(xgb, params, d, 3, xgb_model=path)
    ma, mb = _be().booster_export_model(a.handle), _be().booster_export_model(resumed.handle)
    assert_same_structure(mb, ma)
    assert _same_bits(ma["split_cond"], mb["split_cond"])


WORKER = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import sagemaker_xgboost_container_b200 as xgb
from util import synth
X, y = synth(40000, 12, 52, "multi", K=3)
d = xgb.DMatrix(X, label=y)
b = xgb.train(dict(objective="multi:softprob", num_class=3, subsample=0.3, sampling_method="gradient_based", seed=3, max_depth=6), d,
              num_boost_round=4, verbose_eval=False)
open(sys.argv[2], "wb").write(bytes(b.save_raw("ubj")))
"""


def test_graph_replay_matches_direct_launches(xgb, tmp_path):
    outs = []
    for tag, env_extra in (("graph", {}), ("direct", {"B200XGB_NO_GRAPH": "1"})):
        env = dict(os.environ)
        env.pop("B200XGB_NO_GRAPH", None)
        env.update(env_extra)
        out = str(tmp_path / (tag + ".ubj"))
        r = subprocess.run([sys.executable, "-c", WORKER, ROOT, out], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1]


@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic", "reg:absoluteerror"])
def test_no_change_without_sampling(xgb, objective):
    X, y = synth(30000, 10, 53, "bin" if "logistic" in objective else "reg")
    d = xgb.DMatrix(X, label=y)
    params = dict(objective=objective, max_depth=6, seed=3)
    a = _train(xgb, dict(params, sampling_method="uniform"), d, 4)
    b = _train(xgb, dict(params, sampling_method="gradient_based"), d, 4)
    c = _train(xgb, params, d, 4)
    assert _bytes(a) == _bytes(b) == _bytes(c)


# ---------------------------------------------------------------------------------------------------------------- accuracy
def _logloss(p, y):
    p = np.clip(p.astype(np.float64), 1e-15, 1 - 1e-15)
    return float(-np.mean(y * np.log(p) + (1 - y) * np.log(1 - p)))


def test_accuracy_at_subsample_0_1(xgb):
    """The config-2 recipe (binary:logistic, 28 features, 256 bins) at 1M rows and subsample 0.1 on three seeds: both sampling
    methods train a model whose validation logloss is finite and well below the constant prediction's.  Which of the two ends
    closer to the unsampled model is printed, not asserted: on this data gradient-based sampling did not end closer than uniform
    sampling on the first seed (DESIGN.md, Gradient-based sampling)."""
    for seed in (1, 2, 3):
        X, y = synth(1_200_000, 28, 100 + seed, "bin")
        dt, dv = xgb.DMatrix(X[:1_000_000], label=y[:1_000_000]), xgb.DMatrix(X[1_000_000:])
        yv = y[1_000_000:]
        base = dict(objective="binary:logistic", max_depth=6, eta=0.3, max_bin=256, seed=seed)
        loss = {}
        for name, extra in (("full", {}), ("uniform", dict(subsample=0.1)), ("gradient_based", dict(subsample=0.1, sampling_method="gradient_based"))):
            loss[name] = _logloss(_train(xgb, dict(base, **extra), dt, 60).predict(dv), yv)
        print("seed %d validation logloss: %s" % (seed, json.dumps(loss)))
        const = _logloss(np.full(len(yv), yv.mean()), yv)
        for name in ("uniform", "gradient_based"):
            assert np.isfinite(loss[name]) and loss[name] < loss["full"] + 0.5 * (const - loss["full"]), (seed, loss, const)


# ---------------------------------------------------------------------------------------------------------------- the Python surface
def test_container_string_hyperparameters(xgb):
    X, y = synth(20000, 8, 61, "bin")
    d = xgb.DMatrix(X, label=y)
    hp = {"objective": "binary:logistic", "max_depth": "5", "eta": "0.3", "sampling_method": "gradient_based", "subsample": "0.3"}
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        bst = xgb.train(hp, d, num_boost_round=3, verbose_eval=False)
    cfg = json.loads(bst.save_config())["learner"]["gradient_booster"]["tree_train_param"]
    assert cfg["sampling_method"] == "gradient_based"
    uni = json.loads(_train(xgb, {"objective": "binary:logistic"}, d, 1).save_config())
    assert uni["learner"]["gradient_booster"]["tree_train_param"]["sampling_method"] == "uniform"
    # a pickled booster continues with the same sampling
    full = _train(xgb, hp, d, 5)
    resumed = pickle.loads(pickle.dumps(_train(xgb, hp, d, 2)))
    for r in range(2, 5):
        resumed.update(d, r)
    assert _bytes(resumed) == _bytes(full)


def test_bad_value_raises(xgb):
    X, y = synth(500, 4, 62, "reg")
    with pytest.raises(xgb.core.XGBoostError, match="sampling_method"):
        _train(xgb, dict(objective="reg:squarederror", subsample=0.5, sampling_method="goss"), xgb.DMatrix(X, label=y), 1)
