"""GPU parity tests (run with `pytest -m gpu` on an H100): the CUDA path through the C-ABI against the CPU oracle.

Bar (BASELINE.json north_star): integer work bit-exact (bins, fixed-point histograms, leaf indices, tree structure);
leaf weights within 1e-5 of the CPU reference.
"""
import numpy as np
import pytest

from util import assert_same_structure, first_structural_difference, max_leaf_diff, synth

pytestmark = pytest.mark.gpu

LEAF_TOL = 1e-5       # absolute, stated by BASELINE.json north_star
MARGIN_TOL = 2e-5


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


@pytest.mark.parametrize("n,F,max_bin,quantised", [(5000, 7, 256, True), (20000, 28, 256, True), (3000, 5, 64, False), (4000, 40, 256, False)])
def test_cuts_and_bins_match_oracle(xgb, oracle, n, F, max_bin, quantised):
    X, y = synth(n, F, 11, "reg", quantised=quantised)
    d = xgb.DMatrix(X, label=y)
    ptrs, vals, mins, hm = _be().dmatrix_get_cuts(d.handle, max_bin)
    optrs, ovals, omins, ohm = oracle.make_cuts(X, max_bin)
    np.testing.assert_array_equal(ptrs, optrs)
    np.testing.assert_array_equal(vals, ovals)
    np.testing.assert_array_equal(mins, omins)
    assert hm == ohm
    bins = _be().dmatrix_get_bins(d.handle, max_bin)
    np.testing.assert_array_equal(bins, oracle.bin_matrix(X, optrs, ovals))      # bit-exact integer work


def test_bins_with_missing_values(xgb, oracle):
    X, y = synth(6000, 9, 12, "reg", quantised=False, missing_frac=0.1)
    d = xgb.DMatrix(X, label=y)
    ptrs, vals, mins, hm = _be().dmatrix_get_cuts(d.handle, 256)
    optrs, ovals, omins, ohm = oracle.make_cuts(X, 256)
    assert hm and ohm
    np.testing.assert_array_equal(ptrs, optrs)
    np.testing.assert_array_equal(vals, ovals)
    np.testing.assert_array_equal(_be().dmatrix_get_bins(d.handle, 256), oracle.bin_matrix(X, optrs, ovals))


HIST_SHAPES = [(1, 3), (17, 5), (4096, 28), (4097, 33), (100003, 50), (300000, 100), (70001, 36), (50000, 104), (20000, 130)]
MODE_KERNEL = {0: "hist_root_kernel<GH>", 1: "hist_gather_kernel", 2: "hist_root_kernel<GONLY>"}


def _hist_inputs(xgb, n, F, seed=21):
    X, y = synth(n, F, seed, "reg")
    rng = np.random.default_rng(5)
    gpair = np.stack([rng.standard_normal(n).astype(np.float32) * 3, rng.random(n).astype(np.float32) + 0.01], axis=1)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster({"max_bin": 256}, [d])
    return X, gpair, d, b


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n,F", HIST_SHAPES)
def test_root_histogram_bit_exact(xgb, oracle, n, F, mode):
    """Both histogram kernels (TMA-staged root kernel incl. its G-only variant, gather kernel) vs the fixed-point mirror
    in the oracle: exact int64 equality for ragged sizes and every feature layout (padded group, 4- and 8-wide tails,
    two group chunks)."""
    X, gpair, d, b = _hist_inputs(xgb, n, F)
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gpair, mode=mode)
    # 3 groups of G+H planes (192 KB) leave no room for a useful TMA ring: those shapes use the gather kernel for their root pass too
    assert kernel == MODE_KERNEL[mode] or (mode == 0 and F in (100, 104) and kernel == "hist_gather_kernel")
    gq = np.rint(gpair[:, 0] * scales[0]).astype(np.int32)
    hq = np.rint(gpair[:, 1] * scales[1]).astype(np.int32)
    bins = _be().dmatrix_get_bins(d.handle, 256)
    ref = oracle.build_hist_fixed(bins, gq, hq)
    if mode == 2:                      # constant-hessian fast path: only G is accumulated, the H plane is pre-loaded by the caller
        np.testing.assert_array_equal(hist[:, :, 0], ref[:, :, 0])
        assert not hist[:, :, 1].any()
        return
    np.testing.assert_array_equal(hist, ref)
    # and close to the reference-faithful double histogram (same bins, float gradients)
    optrs, ovals, _, _ = oracle.make_cuts(X, 256)
    dref = oracle.build_hist(bins, optrs, gpair)
    for f in range(F):
        nb = optrs[f + 1] - optrs[f]
        got = hist[f, :nb, 0] / scales[0]
        np.testing.assert_allclose(got, dref[optrs[f]:optrs[f + 1], 0], rtol=0, atol=2e-5 * max(1.0, np.abs(gpair[:, 0]).max()) * np.sqrt(n))


@pytest.mark.parametrize("tail_by_position", [False, True])
@pytest.mark.parametrize("n,F,frac,ordered", [(50000, 28, 0.3, True), (120000, 100, 0.25, True), (30000, 50, 0.5, False), (40000, 130, 0.1, True), (9000, 40, 1.0, False)])
def test_gathered_histogram_bit_exact(xgb, oracle, n, F, frac, ordered, tail_by_position):
    """The deeper levels' access pattern: a row subset by row id (ascending like a partitioned node, or shuffled), gradient
    pairs by position."""
    X, gpair, d, b = _hist_inputs(xgb, n, F, seed=23)
    rng = np.random.default_rng(9)
    m = max(1, int(n * frac))
    rows = rng.choice(n, size=m, replace=False).astype(np.uint32)
    if ordered:
        rows.sort()
    gp_pos = gpair[:m]
    # mode 4: the rows' 4 tail bytes are supplied by position, as after a partition (the training path); 0: gathered from bins_tail
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gp_pos, mode=4 if tail_by_position else 0, row_ids=rows)
    assert kernel == "hist_gather_kernel"
    gq = np.zeros(n, np.int32); hq = np.zeros(n, np.int32)
    gq[rows] = np.rint(gp_pos[:, 0] * scales[0]).astype(np.int32)
    hq[rows] = np.rint(gp_pos[:, 1] * scales[1]).astype(np.int32)
    bins = _be().dmatrix_get_bins(d.handle, 256)
    np.testing.assert_array_equal(hist, oracle.build_hist_fixed(bins, gq, hq, rows=rows))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_histogram_int32_overflow_spill_path(xgb, oracle, mode):
    """2.4 M rows x 100 features with a constant column, a 95 %-skewed column and same-sign gradients near the top of the
    fixed-point grid: every CTA crosses several 8064-row windows and its hot accumulators pass 2^24 in each of them, so the
    sparse RED.ADD.64 spill between windows carries most of the mass.  Bit-exact against the oracle's int64 mirror."""
    n, F = 2_400_000, 100
    rng = np.random.default_rng(77)
    X = rng.integers(0, 200, size=(n, F)).astype(np.float32)
    X[:, 0] = 3.0                                              # constant column: one bin takes every row
    X[:, 1] = np.where(rng.random(n) < 0.95, 7.0, X[:, 1])     # heavily skewed column
    X[:, 97] = 1.0                                             # constant column in the narrow tail block
    gpair = np.stack([(0.6 + 0.4 * rng.random(n)).astype(np.float32) * 5, (0.5 + 0.5 * rng.random(n)).astype(np.float32)], axis=1)
    d = xgb.DMatrix(X, label=np.zeros(n, np.float32))
    b = xgb.Booster({"max_bin": 256}, [d])
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gpair, mode=mode)
    gq = np.rint(gpair[:, 0] * scales[0]).astype(np.int32)
    hq = np.rint(gpair[:, 1] * scales[1]).astype(np.int32)
    assert gq.min() > (1 << 16) and int(gq.astype(np.int64).sum()) > (1 << 38)       # the window sums really exceed int32 many times over
    bins = _be().dmatrix_get_bins(d.handle, 256)
    ref = oracle.build_hist_fixed(bins, gq, hq)
    np.testing.assert_array_equal(hist[:, :, 0], ref[:, :, 0])
    if mode != 2:
        np.testing.assert_array_equal(hist[:, :, 1], ref[:, :, 1])


CASES = [
    ("reg:squarederror", "reg", 1, dict(max_depth=6, eta=0.3), 20000, 28, 12),
    ("reg:squarederror", "reg", 1, dict(max_depth=5, eta=0.2, gamma=4, min_child_weight=6), 3000, 8, 20),
    ("binary:logistic", "bin", 1, dict(max_depth=6, eta=0.3), 30000, 28, 12),
    ("binary:logistic", "bin", 1, dict(max_depth=4, eta=0.1, alpha=0.5, scale_pos_weight=2.0), 10000, 40, 10),
    ("multi:softprob", "multi", 4, dict(max_depth=4, eta=0.3), 12000, 20, 5),
    ("reg:squarederror", "reg", 1, dict(max_depth=3, eta=0.5, max_delta_step=0.7), 5000, 100, 6),
    ("binary:logistic", "bin", 1, dict(max_depth=5, eta=0.3), 40000, 100, 6),      # 3 groups + tail with G and H: 192 KB of planes, the root pass runs in the gather kernel
]


@pytest.mark.parametrize("objective,kind,K,hp,n,F,rounds", CASES)
def test_training_matches_oracle(xgb, oracle, objective, kind, K, hp, n, F, rounds):
    X, y = synth(n, F, 31, kind, K=max(K, 1))
    params = dict(objective=objective, tree_method="hist", max_bin=256, **hp)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    ref = oracle.train(params, X, y, rounds)
    mr = ref.model()
    assert abs(m["base_score"] - mr["base_score"]) <= 1e-6 * max(1.0, abs(mr["base_score"]))
    assert first_structural_difference(m, mr) is None, "tree structure differs first at tree %s" % first_structural_difference(m, mr)
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    # prediction cache kept by the trainer == oracle margins
    cache = _be().booster_cached_margin(bst.handle, d.handle, max(K, 1))
    np.testing.assert_allclose(cache, ref.margins(), rtol=0, atol=MARGIN_TOL)
    # predict(): leaf indices are integer work -> bit-exact against the oracle walking ITS model
    leaves = bst.predict(d, pred_leaf=True)
    np.testing.assert_array_equal(leaves.astype(np.int32), oracle.predict_leaf(mr, X))
    margin = bst.predict(d, output_margin=True).reshape(n, -1)
    np.testing.assert_allclose(margin, oracle.predict_margin(mr, X), rtol=0, atol=MARGIN_TOL)
    # the predictor alone: bit-exact against the oracle walking the model the device exported (MARGIN_TOL above covers
    # the leaf values the two trainers round differently)
    m["objective"] = objective
    np.testing.assert_array_equal(margin.view(np.uint32), oracle.predict_margin(m, X).view(np.uint32))


@pytest.mark.parametrize("hp", [dict(colsample_bytree=0.5), dict(colsample_bylevel=0.5), dict(colsample_bynode=0.3),
                                dict(colsample_bytree=0.8, colsample_bylevel=0.7, colsample_bynode=0.6, subsample=0.8)])
def test_column_and_row_sampling_match_the_oracle(xgb, oracle, hp):
    """colsample_bytree / bylevel / bynode (nested like upstream's ColumnSampler, counter-based RNG shared with the oracle) and
    subsample: same trees as the oracle, and the sampled models really differ from the unsampled one."""
    X, y = synth(20000, 40, 35, "reg")
    params = dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256, seed=11, **hp)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=6, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, 6).model()
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    plain = oracle.train(dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=256, seed=11), X, y, 6).model()
    assert not np.array_equal(plain["split_index"], mr["split_index"])
    cfg = __import__("json").loads(bst.save_config())["learner"]["gradient_booster"]["tree_train_param"]
    for k, v in hp.items():
        assert abs(float(cfg[k]) - v) < 1e-6                      # applied values are echoed by save_config


def test_logitraw_with_minority_positive_class(xgb, oracle):
    """binary:logitraw with mean(y) < 0.5 (ADVICE r1): the estimated base score must give a finite base margin (the stump
    weight), trees must split, and the model must match the oracle."""
    X, y = synth(20000, 12, 33, "bin")
    y = (y * (np.random.default_rng(1).random(len(y)) < 0.55)).astype(np.float32)          # ~27 % positives
    assert 0.2 < y.mean() < 0.35
    params = dict(objective="binary:logitraw", max_depth=4, eta=0.3, max_bin=256)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=6, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, 6).model()
    assert 0.0 < m["base_score"] < 0.5 and abs(m["base_score"] - mr["base_score"]) < 1e-6
    assert_same_structure(m, mr)
    assert (m["left"] != -1).sum() > 6 and max_leaf_diff(m, mr) <= LEAF_TOL
    margin = bst.predict(d, output_margin=True)
    assert np.isfinite(margin).all()
    np.testing.assert_allclose(margin.reshape(len(y), -1), oracle.predict_margin(mr, X), rtol=0, atol=MARGIN_TOL)


@pytest.mark.parametrize("objective,kind,K,n,F,rounds", [
    ("reg:squarederror", "reg", 1, 2_000_000, 100, 3),       # BASELINE config 3 family (3 groups + tail, 18-bit grid, several overflow windows per CTA)
    ("binary:logistic", "bin", 1, 1_500_000, 28, 3),         # config 2 family
    ("multi:softprob", "multi", 10, 600_000, 50, 2),         # config 4 family: 10 classes
])
def test_full_model_parity_at_baseline_shape_families(xgb, oracle, objective, kind, K, n, F, rounds):
    """Whole-model parity on the BASELINE.json shapes at the largest size the oracle finishes in about a minute: max_depth 6,
    256 bins, structure identical, leaves within 1e-5, pred_leaf bit-exact."""
    X, y = synth(n, F, 77, kind, K=max(K, 1))
    params = dict(objective=objective, tree_method="hist", max_depth=6, max_bin=256, eta=0.3)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert len(m["tree_info"]) == rounds * max(K, 1)
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    sub = np.arange(0, n, 97)
    np.testing.assert_array_equal(bst.predict(xgb.DMatrix(X[sub]), pred_leaf=True).astype(np.int32), oracle.predict_leaf(mr, X[sub]))


def test_training_with_missing_values(xgb, oracle):
    X, y = synth(15000, 12, 41, "reg", quantised=False, missing_frac=0.15)
    params = dict(objective="reg:squarederror", max_depth=5, eta=0.3, max_bin=64)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=8, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, 8).model()
    assert_same_structure(m, mr)
    assert m["default_left"].sum() > 0          # the backward scan was exercised
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    np.testing.assert_array_equal(bst.predict(d, pred_leaf=True).astype(np.int32), oracle.predict_leaf(mr, X))


def test_fixture_model_predict_leaf_bit_exact(xgb, oracle):
    """The reference's own UBJSON fixture through the C++ loader + GPU predictor vs the oracle walking the same file."""
    import os
    from oracle import ubjson
    path = os.path.join(os.path.dirname(__file__), "golden", "abalone_xgboost-model.ubj")
    bst = xgb.Booster(model_file=path)
    mr = ubjson.model_from_xgb_json(ubjson.load(path))
    rng = np.random.default_rng(3)
    X = rng.random((2000, 8)).astype(np.float32) * np.array([3, 1, 1, 0.3, 3, 1.5, 0.8, 1], np.float32)
    X[0] = [2, 0.645, 0.515, 0.15, 1.212, 0.515, 0.2055, 0.385]      # LIBSVM_SAMPLE of test/integration/local/test_abalone.py:24
    d = xgb.DMatrix(X)
    leaves = bst.predict(d, pred_leaf=True).astype(np.int32)
    np.testing.assert_array_equal(leaves, oracle.predict_leaf(mr, X))
    np.testing.assert_array_equal(leaves[0, :8], [42, 45, 40, 43, 34, 38, 38, 41])          # SURVEY.md 8(c) self-consistency vector
    pred = bst.predict(d)
    np.testing.assert_allclose(pred, oracle.predict_margin(mr, X)[:, 0], rtol=0, atol=1e-5)
    assert abs(float(pred[0]) - 11.100031) < 1e-4


def test_model_roundtrip_ubj_json_pickle(xgb, oracle, tmp_path):
    import pickle
    from oracle import ubjson
    X, y = synth(4000, 10, 51, "bin")
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(objective="binary:logistic", max_depth=4), d, num_boost_round=5, verbose_eval=False)
    p0 = bst.predict(d)
    f_ubj, f_json = str(tmp_path / "xgboost-model"), str(tmp_path / "m.json")
    bst.save_model(f_ubj)
    bst.save_model(f_json)
    for f in (f_ubj, f_json):
        b2 = xgb.Booster(model_file=f)
        np.testing.assert_array_equal(b2.predict(d), p0)
    b3 = pickle.loads(pickle.dumps(bst))
    np.testing.assert_array_equal(b3.predict(d), p0)
    # the independent Python reader understands the C++ writer's UBJSON
    doc = ubjson.load(f_ubj)
    mo = ubjson.model_from_xgb_json(doc)
    assert mo["objective"] == "binary:logistic" and len(mo["tree_info"]) == 5
    np.testing.assert_allclose(oracle.transform(mo, oracle.predict_margin(mo, X))[:, 0], p0, rtol=0, atol=1e-6)
    cfg = __import__("json").loads(bst.save_config())
    assert cfg["learner"]["objective"]["name"] == "binary:logistic"


def test_continue_training_from_checkpoint(xgb, oracle, tmp_path):
    X, y = synth(6000, 9, 61, "reg")
    params = dict(objective="reg:squarederror", max_depth=4, eta=0.3)
    d = xgb.DMatrix(X, label=y)
    full = xgb.train(params, d, num_boost_round=8, verbose_eval=False)
    part = xgb.train(params, d, num_boost_round=5, verbose_eval=False)
    ck = str(tmp_path / "xgboost-checkpoint.4")
    part.save_model(ck)
    resumed = xgb.train(params, d, num_boost_round=3, xgb_model=ck, verbose_eval=False)
    assert resumed.num_boosted_rounds() == 8
    np.testing.assert_allclose(resumed.predict(d), full.predict(d), rtol=0, atol=1e-5)


def test_eval_metrics_match_numpy(xgb):
    X, y = synth(5000, 6, 71, "bin")
    d = xgb.DMatrix(X, label=y)
    res = {}
    bst = xgb.train(dict(objective="binary:logistic", max_depth=3, eval_metric=["logloss", "error", "rmse"]), d, num_boost_round=3,
                    evals=[(d, "train")], evals_result=res, verbose_eval=False)
    p = bst.predict(d).astype(np.float64)
    ll = -np.mean(y * np.log(p) + (1 - y) * np.log(1 - p))
    assert abs(res["train"]["logloss"][-1] - ll) < 1e-6
    assert abs(res["train"]["error"][-1] - np.mean((p > 0.5) != (y > 0.5))) < 1e-9
    assert abs(res["train"]["rmse"][-1] - np.sqrt(np.mean((p - y) ** 2))) < 1e-6


MORE_OBJECTIVES = [
    ("reg:squaredlogerror", "pos", {}, "rmsle"),
    ("reg:pseudohubererror", "reg", dict(huber_slope=0.7), "mphe"),
    ("count:poisson", "count", {}, "poisson-nloglik"),
    ("count:poisson", "count", dict(max_delta_step=0.3), "poisson-nloglik"),
    ("reg:gamma", "pos", {}, "gamma-nloglik"),
    ("reg:tweedie", "count", dict(tweedie_variance_power=1.3), "tweedie-nloglik@1.3"),
    ("binary:hinge", "bin", {}, "error"),
]


def _numpy_metric(name, y, p, slope=1.0):
    y = y.astype(np.float64); p = p.astype(np.float64)
    if name == "rmsle":
        return np.sqrt(np.mean((np.log1p(y) - np.log1p(p)) ** 2))
    if name == "mape":
        return np.mean(np.abs((y - p) / y))
    if name == "mphe":
        return np.mean(slope ** 2 * (np.sqrt(1 + ((y - p) / slope) ** 2) - 1))
    if name == "poisson-nloglik":
        from scipy.special import gammaln
        p = np.maximum(p, 1e-16)
        return np.mean(gammaln(y + 1) + p - np.log(p) * y)
    if name == "gamma-nloglik":
        p = np.maximum(p, 1e-6)
        return np.mean(y / p + np.log(p))
    if name == "gamma-deviance":
        return 2 * np.mean(np.log((p + 1e-6) / (y + 1e-6)) + (y + 1e-6) / (p + 1e-6) - 1)
    if name.startswith("tweedie-nloglik@"):
        rho = float(name.split("@")[1])
        return np.mean(-y * np.exp((1 - rho) * np.log(p)) / (1 - rho) + np.exp((2 - rho) * np.log(p)) / (2 - rho))
    if name == "error":
        return np.mean((p > 0.5) != (y > 0.5))
    raise ValueError(name)


@pytest.mark.parametrize("objective,kind,hp,default_metric", MORE_OBJECTIVES)
def test_remaining_elementwise_objectives_match_oracle(xgb, oracle, objective, kind, hp, default_metric):
    """The other element-wise objectives the container's hyperparameter validation accepts (hyperparameter_validation.py:283-309):
    gradients, base score, prediction transform, default metric name and value."""
    n, F, rounds = 8000, 12, 6
    X, y = synth(n, F, 57, kind)
    params = dict(objective=objective, tree_method="hist", max_depth=4, eta=0.3, **hp)
    d = xgb.DMatrix(X, label=y)
    res = {}
    bst = xgb.train(params, d, num_boost_round=rounds, evals=[(d, "train")], evals_result=res, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert abs(m["base_score"] - mr["base_score"]) <= 1e-6 * max(1.0, abs(mr["base_score"]))
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    margin = bst.predict(d, output_margin=True)
    np.testing.assert_allclose(margin, oracle.predict_margin(mr, X).ravel(), rtol=0, atol=MARGIN_TOL)
    pred = bst.predict(d)
    np.testing.assert_allclose(pred, oracle.transform(mr, oracle.predict_margin(mr, X)).ravel(), rtol=2e-6, atol=1e-6)
    assert list(res["train"].keys()) == [default_metric]                       # the objective's default metric, upstream's spelling
    ref = _numpy_metric(default_metric, y, pred, slope=hp.get("huber_slope", 1.0))
    assert abs(res["train"][default_metric][-1] - ref) <= 2e-5 * max(1.0, abs(ref))
    # the objective's parameters survive save_config / load_config and a model round trip
    cfg = bst.save_config()
    b2 = xgb.Booster(model_file=bytes(bst.save_raw("ubj")))
    b2.load_config(cfg)
    np.testing.assert_array_equal(b2.predict(d), pred)


def test_extra_metrics_and_label_checks_of_the_new_objectives(xgb):
    X, y = synth(4000, 6, 58, "pos")
    d = xgb.DMatrix(X, label=y)
    res = {}
    bst = xgb.train(dict(objective="reg:gamma", max_depth=3, eval_metric=["gamma-deviance", "mape", "rmsle", "mphe", "gamma-nloglik"]), d, num_boost_round=4,
                    evals=[(d, "train")], evals_result=res, verbose_eval=False)
    p = bst.predict(d)
    for name in ("gamma-deviance", "mape", "rmsle", "mphe", "gamma-nloglik"):
        ref = _numpy_metric(name, y, p)
        assert abs(res["train"][name][-1] - ref) <= 2e-5 * max(1.0, abs(ref)), name
    for objective, bad, msg in (("count:poisson", -1.0, "label must be nonnegative"), ("reg:gamma", 0.0, "label must be positive"),
                                ("reg:tweedie", -0.5, "label must be nonnegative"), ("reg:squaredlogerror", -1.0, "label must be greater than -1")):
        yb = y.copy(); yb[3] = bad
        with pytest.raises(xgb.XGBoostError, match=msg):
            xgb.train(dict(objective=objective), xgb.DMatrix(X, label=yb), num_boost_round=1, verbose_eval=False)


@pytest.mark.parametrize("objective,kind,K,missing", [("reg:squarederror", "reg", 1, 0.0), ("binary:logistic", "bin", 1, 0.15), ("multi:softprob", "multi", 3, 0.0)])
def test_pred_contribs_are_the_exact_shapley_values(xgb, oracle, objective, kind, K, missing):
    """Booster.predict(pred_contribs=True) (test_abalone.py:65): the device Tree SHAP against brute-force Shapley values of the
    cover-weighted game (oracle.shap_bruteforce enumerates all 2^F feature subsets), incl. missing values, several classes and
    iteration_range; the contributions of a row add up to its margin."""
    n, F, rounds = 400, 8, 6
    X, y = synth(n, F, 63, kind, K=max(K, 1), missing_frac=missing)
    params = dict(objective=objective, max_depth=4, eta=0.4)
    if K > 1:
        params["num_class"] = K
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    m["objective"] = objective                      # the oracle derives the base margin (logit of base_score, ...) from it
    phi = bst.predict(d, pred_contribs=True)
    assert phi.shape == ((n, F + 1) if K == 1 else (n, K, F + 1))
    ref = oracle.shap_bruteforce(m, X)
    np.testing.assert_allclose(phi.reshape(n, max(K, 1), F + 1), ref, rtol=0, atol=2e-5)
    np.testing.assert_allclose(phi.reshape(n, max(K, 1), F + 1).sum(-1), bst.predict(d, output_margin=True).reshape(n, -1), rtol=0, atol=2e-5)
    part = bst.predict(d, pred_contribs=True, iteration_range=(1, 4))
    np.testing.assert_allclose(part.reshape(n, max(K, 1), F + 1), oracle.shap_bruteforce(m, X, tree_begin=1 * max(K, 1), tree_end=4 * max(K, 1)), rtol=0, atol=2e-5)


def test_pred_contribs_add_up_to_the_margin_on_a_wide_deep_model(xgb):
    n, F = 3000, 60
    X, y = synth(n, F, 64, "reg", missing_frac=0.05)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(max_depth=9, eta=0.2, min_child_weight=1), d, num_boost_round=8, verbose_eval=False)
    phi = bst.predict(d, pred_contribs=True)
    assert phi.shape == (n, F + 1)
    np.testing.assert_allclose(phi.sum(1), bst.predict(d, output_margin=True), rtol=0, atol=1e-4)
    with pytest.raises(xgb.XGBoostError, match="not implemented"):
        bst.predict(d, pred_interactions=True)


@pytest.mark.parametrize("hp,objective,kind,n,F", [
    (dict(max_leaves=16, max_depth=0), "reg:squarederror", "reg", 20000, 28),
    (dict(max_leaves=0, max_depth=4), "reg:squarederror", "reg", 8000, 100),       # bounded by depth only: ends as a full tree
    (dict(max_leaves=12, max_depth=3, gamma=2.0), "binary:logistic", "bin", 15000, 12),   # a top candidate at max_depth ends the tree early
    (dict(max_leaves=40, max_depth=0, min_child_weight=5, eta=0.2), "binary:logistic", "bin", 30000, 40),
])
def test_lossguide_growth_matches_oracle(xgb, oracle, hp, objective, kind, n, F):
    """grow_policy=lossguide (hyperparameter_validation.py accepts it with max_leaves): best-first expansion, one node per
    iteration, node ids in expansion order -- structure, leaf values and pred_leaf against the oracle's restatement of
    upstream's loss-guided Driver."""
    rounds = 5
    X, y = synth(n, F, 97, kind)
    params = dict(dict(objective=objective, tree_method="hist", grow_policy="lossguide", eta=0.3), **hp)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    if hp["max_leaves"]:
        leaves = [int((m["left"][a:b] == -1).sum()) for a, b in zip(m["tree_offset"][:-1], m["tree_offset"][1:])]
        assert max(leaves) <= hp["max_leaves"]
    np.testing.assert_array_equal(bst.predict(d, pred_leaf=True).astype(np.int32), oracle.predict_leaf(mr, X))
    np.testing.assert_allclose(bst.predict(d, output_margin=True), oracle.predict_margin(mr, X).ravel(), rtol=0, atol=MARGIN_TOL)
    m["objective"] = objective
    np.testing.assert_array_equal(bst.predict(d, output_margin=True).view(np.uint32), oracle.predict_margin(m, X).ravel().view(np.uint32))
    if hp["max_leaves"] == 40:          # best-first growth stops at 40 leaves: not a level-complete tree
        assert max(leaves) == 40
        t0 = slice(m["tree_offset"][0], m["tree_offset"][1])
        depth = np.zeros(t0.stop - t0.start, int)
        for i, p in enumerate(m["parent"][t0]):
            if i:
                depth[i] = depth[p] + 1
        leaf_depths = depth[m["left"][t0] == -1]
        assert leaf_depths.max() > leaf_depths.min()


@pytest.mark.parametrize("extra", [dict(max_depth=5), dict(max_depth=4, alpha=0.3, max_delta_step=0.5), dict(grow_policy="lossguide", max_leaves=20, max_depth=0)])
def test_monotone_constraints_match_oracle_and_hold(xgb, oracle, extra):
    """monotone_constraints (hyperparameter_validation.py passes the tuple through): clamped weights, gain at the clamped weights,
    rejected violating candidates, bounds handed to the children -- same trees as the oracle's restatement of upstream's
    TreeEvaluator, and the fitted function really is monotone in the constrained features."""
    n, F, rounds = 20000, 6, 8
    rng = np.random.default_rng(12)
    X, _ = synth(n, F, 12, "reg")
    y = (np.sin(2 * X[:, 0]) + 0.5 * X[:, 1] - X[:, 2] ** 2 + 0.2 * rng.standard_normal(n)).astype(np.float32)
    cons = (1, -1, 0, 0, 0, 0)
    params = dict(dict(objective="reg:squarederror", eta=0.3, monotone_constraints=cons), **extra)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    for f, sign in ((0, 1), (1, -1)):
        for trial in range(20):
            grid = np.tile(X[rng.integers(n)], (128, 1)).astype(np.float32)
            grid[:, f] = np.linspace(-3.5, 3.5, 128, dtype=np.float32)
            p = bst.predict(xgb.DMatrix(grid), output_margin=True)
            assert np.all(sign * np.diff(p) >= -1e-6), "feature %d is not monotone" % f
    assert "monotone_constraints" in bst.save_config()
    # the unconstrained fit is NOT monotone in feature 0 (sin): the constraint did something
    free = xgb.train(dict(objective="reg:squarederror", eta=0.3, max_depth=5), d, num_boost_round=rounds, verbose_eval=False)
    grid = np.tile(np.median(X, 0), (128, 1)).astype(np.float32); grid[:, 0] = np.linspace(-3.5, 3.5, 128, dtype=np.float32)
    assert np.any(np.diff(free.predict(xgb.DMatrix(grid), output_margin=True)) < -1e-3)


def _paths_respect(model, groups):
    """every root-to-leaf path uses features of ONE constraint set (or a single feature outside every set)"""
    for t in range(len(model["tree_info"])):
        a, b = model["tree_offset"][t], model["tree_offset"][t + 1]
        left, right, si = model["left"][a:b], model["right"][a:b], model["split_index"][a:b]
        stack = [(0, frozenset())]
        while stack:
            i, feats = stack.pop()
            if left[i] == -1:
                if len(feats) > 1 and not any(feats <= set(g) for g in groups):
                    return False
                continue
            f = feats | {int(si[i])}
            stack.append((int(left[i]), f)); stack.append((int(right[i]), f))
    return True


@pytest.mark.parametrize("extra", [dict(max_depth=5), dict(grow_policy="lossguide", max_leaves=24, max_depth=0)])
def test_interaction_constraints_match_oracle_and_hold(xgb, oracle, extra):
    n, F, rounds = 20000, 7, 8
    rng = np.random.default_rng(21)
    X, _ = synth(n, F, 21, "reg")
    y = (X[:, 0] * X[:, 1] + X[:, 2] * X[:, 3] + X[:, 4] + 0.5 * X[:, 5] * X[:, 0] + 0.1 * rng.standard_normal(n)).astype(np.float32)
    groups = [[0, 1], [2, 3, 4]]                                    # features 5 and 6 are in no set
    params = dict(dict(objective="reg:squarederror", eta=0.3, interaction_constraints=groups), **extra)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert first_structural_difference(m, mr) is None
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    assert _paths_respect(m, groups)
    free_bst = xgb.train(dict(objective="reg:squarederror", eta=0.3, max_depth=5), d, num_boost_round=rounds, verbose_eval=False)
    free = _be().booster_export_model(free_bst.handle)              # (keep the Booster alive: its handle dies with it)
    assert not _paths_respect(free, groups)                         # the unconstrained trees do mix the sets
    assert "interaction_constraints" in bst.save_config()


@pytest.mark.parametrize("weighted", [False, True])
def test_auc_matches_sklearn(xgb, weighted):
    """Native `auc` (the one HPO metric the container does not compute itself, train_utils.py:45-76) against
    sklearn.metrics.roc_auc_score, with tied predictions (shallow trees give few distinct scores) and sample weights."""
    from sklearn.metrics import roc_auc_score
    X, y = synth(30000, 10, 91, "bin")
    w = np.random.default_rng(4).random(len(y)).astype(np.float32) + 0.1 if weighted else None
    d = xgb.DMatrix(X, label=y, weight=w)
    res = {}
    bst = xgb.train(dict(objective="binary:logistic", max_depth=2, eta=0.5, eval_metric=["auc", "logloss"]), d, num_boost_round=3,
                    evals=[(d, "train")], evals_result=res, verbose_eval=False)
    p = bst.predict(d)
    assert len(np.unique(p)) < 200                                   # many ties
    assert abs(res["train"]["auc"][-1] - roc_auc_score(y, p, sample_weight=w)) < 1e-9


def test_label_errors_surface_as_xgboost_error(xgb):
    X, y = synth(200, 4, 81, "reg")
    d = xgb.DMatrix(X, label=y * 10)
    with pytest.raises(xgb.XGBoostError, match=r"label must be in \[0,1\] for logistic regression"):
        xgb.train(dict(objective="binary:logistic"), d, num_boost_round=1, verbose_eval=False)
    d2 = xgb.DMatrix(X, label=np.full(200, 7, np.float32))
    with pytest.raises(xgb.XGBoostError, match=r"label must be in \[0, num_class\)"):
        xgb.train(dict(objective="multi:softprob", num_class=3), d2, num_boost_round=1, verbose_eval=False)
