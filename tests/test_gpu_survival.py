"""survival:aft and survival:cox on the GPU: gradients against tests/survival_reference.py through
XGB200BoosterComputeGradient, trees against the oracle's trainer on the survival gradients, the metrics, determinism of the
Cox scans, serving and model IO, the container's string hyperparameters, dart / forests, and the errors."""
import json
import os
import pickle

import numpy as np
import pytest

import survival_reference as SR
from util import assert_same_structure, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
LEAF_TOL = 1e-5
MARGIN_TOL = 2e-5


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _aft_data(n, F, seed):
    """Features and interval labels with every censoring type: uncensored, right (upper = inf), left (lower = 0), interval."""
    X, y = synth(n, F, seed, "reg")
    rng = np.random.default_rng(seed)
    t = np.exp(1.0 + 0.5 * y + 0.3 * rng.standard_normal(n)).astype(np.float32)
    lo, hi = t.copy(), t.copy()
    kind = rng.integers(0, 4, n)
    hi[kind == 1] = np.inf
    lo[kind == 2] = 0.0
    hi[kind == 3] = (t[kind == 3] * rng.uniform(1.1, 2.5, (kind == 3).sum())).astype(np.float32)
    return X, lo, hi


def _cox_data(n, F, seed, levels=500):
    X, y = synth(n, F, seed, "reg")
    rng = np.random.default_rng(seed)
    t = np.ceil(np.exp(1.0 - 0.5 * y + 0.5 * rng.standard_normal(n)) * levels / 20).astype(np.float32)     # many ties
    return X, np.where(rng.random(n) < 0.7, t, -t).astype(np.float32)


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("dist", ["normal", "logistic", "extreme"])
def test_aft_gradient_matches_reference(xgb, dist):
    n = 20000
    X, lo, hi = _aft_data(n, 4, 1)
    w = np.random.default_rng(2).uniform(0.2, 3.0, n).astype(np.float32)
    d = xgb.DMatrix(X, weight=w, label_lower_bound=lo, label_upper_bound=hi)
    rng = np.random.default_rng(3)
    margins = [np.log(np.where(lo > 0, lo, hi)) + rng.uniform(-2, 2, n), rng.uniform(-40, 40, n), np.full(n, 40.0), np.full(n, -40.0)]
    margins = [m.astype(np.float32) for m in margins]
    for sigma in (0.7, 2.0):
        params = dict(objective="survival:aft", aft_loss_distribution=dist, aft_loss_distribution_scale=sigma)
        bst = xgb.Booster(params, [d])
        for m in margins:
            got = _be().booster_compute_gradient(bst.handle, d.handle, m)[:, 0, :]
            want = SR.aft_gradient(m, lo, hi, w, dist, sigma)
            assert np.all(np.isfinite(got))
            assert np.all((np.abs(got[:, 0]) <= 15 * w) & (got[:, 1] >= np.float32(1e-16) * w * (1 - 1e-6)) & (got[:, 1] <= 15 * w))
            # within 2 float ulps wherever the pair does not hinge on the math library's last bits (see SR.aft_conditioned);
            # near the labels that is every row
            ok = SR.aft_conditioned(m, lo, hi, w, dist, sigma)
            assert ok.mean() > (0.999 if m is margins[0] else 0.4)
            u = _ulps(got, want).max(axis=1)
            if m is margins[0]:
                assert u.max() <= 2, (dist, sigma, int(u.max()), int((u > 2).sum()))
            else:      # far from the labels a few more rows hinge on exp() underflow and limit branches the jitter does not move
                assert (u[ok] <= 2).mean() >= 0.99, (dist, sigma, int((u[ok] > 2).sum()))


def test_cox_gradient_matches_reference_on_3m_rows(xgb):
    n = 3_000_000                       # more scan tiles than one CTA covers, and the 18-bit grid
    X, y = _cox_data(n, 2, 4, levels=20000)
    w = np.random.default_rng(5).uniform(0.5, 2.0, n).astype(np.float32)
    d = xgb.DMatrix(X, label=y, weight=w)
    bst = xgb.Booster(dict(objective="survival:cox"), [d])
    m = np.random.default_rng(6).normal(0, 1, n).astype(np.float32)
    got = _be().booster_compute_gradient(bst.handle, d.handle, m)[:, 0, :]
    # the product sums exp() in double throughout; upstream's float exp() total would move the last rows of the order by
    # its own rounding (survival_reference.cox_gradient), so the comparison isolates suffix sums against running subtraction
    want = SR.cox_gradient(m, y, w, float_total=False)
    for k in (0, 1):
        scale = np.abs(want[:, k]).max()
        np.testing.assert_allclose(got[:, k], want[:, k], rtol=1e-6, atol=1e-6 * scale)


def test_subsample_masks_equal_the_reference(xgb):
    n = 30000
    X, lo, hi = _aft_data(n, 3, 7)
    _, y = _cox_data(n, 3, 7)
    for params, kw in ((dict(objective="survival:aft"), dict(label_lower_bound=lo, label_upper_bound=hi)), (dict(objective="survival:cox"), dict(label=y))):
        params.update(subsample=0.6, seed=9)
        d = xgb.DMatrix(X, **kw)
        bst = xgb.Booster(params, [d])
        m = np.zeros(n, np.float32)
        for rnd in (0, 3):
            got = _be().booster_compute_gradient(bst.handle, d.handle, m, rnd)[:, 0, :]
            keep = SR.sample_mask(n, 9, rnd, 0.6)
            np.testing.assert_array_equal(got[~keep], 0.0)
            assert np.all(got[keep, 1] != 0.0)


TREES = {
    "aft-normal": (dict(objective="survival:aft", aft_loss_distribution="normal", aft_loss_distribution_scale=1.2), False),
    "aft-logistic": (dict(objective="survival:aft", aft_loss_distribution="logistic", aft_loss_distribution_scale=0.8), False),
    "aft-extreme": (dict(objective="survival:aft", aft_loss_distribution="extreme"), False),
    "aft-lossguide": (dict(objective="survival:aft", grow_policy="lossguide", max_leaves=12, max_depth=0), False),
    "cox-ties": (dict(objective="survival:cox"), True),
}


@pytest.mark.parametrize("case", sorted(TREES))
def test_trees_match_the_oracle(xgb, oracle, case):
    extra, cox = TREES[case]
    n = 20000
    params = dict(tree_method="hist", max_bin=256, max_depth=5, eta=0.5, seed=3)
    params.update(extra)
    w = np.random.default_rng(8).uniform(0.5, 2.0, n).astype(np.float32)
    if cox:
        X, y = _cox_data(n, 12, 9)
        d = xgb.DMatrix(X, label=y, weight=w)
        kw = dict(label=y)
    else:
        X, lo, hi = _aft_data(n, 12, 9)
        d = xgb.DMatrix(X, weight=w, label_lower_bound=lo, label_upper_bound=hi)
        kw = dict(lower=lo, upper=hi)
    bst = xgb.Booster(params, [d])
    ref = SR.SurvivalTrainer(params, X, weight=w, bins=_be().dmatrix_get_bins(d.handle, 256), cuts=_be().dmatrix_get_cuts(d.handle, 256), **kw)
    for r in range(4):
        bst.update(d, r)
        ref.update()
    m, mr = _be().booster_export_model(bst.handle), ref.model()
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= LEAF_TOL
    margin = bst.predict(d, output_margin=True).reshape(-1, 1)
    np.testing.assert_allclose(margin, ref.margins(), rtol=0, atol=MARGIN_TOL)
    mm = margin[:, 0]
    line = bst.eval_set([(d, "train")], 4)
    vals = dict(kv.split(":") for kv in line.split("\t")[1:])
    if cox:
        assert float(vals["train-cox-nloglik"]) == pytest.approx(SR.cox_nloglik(mm, y), rel=1e-6)
    else:
        dist, sigma = params.get("aft_loss_distribution", "normal"), float(params.get("aft_loss_distribution_scale", 1.0))
        assert float(vals["train-aft-nloglik"]) == pytest.approx(SR.aft_nloglik(mm, lo, hi, w, dist, sigma), rel=1e-6)
        bst.set_param({"eval_metric": "interval-regression-accuracy"})
        line = bst.eval_set([(d, "train")], 4)
        vals = dict(kv.split(":") for kv in line.split("\t")[1:])
        assert float(vals["train-interval-regression-accuracy"]) == pytest.approx(SR.interval_accuracy(mm, lo, hi, w), rel=1e-6)


def _cox_train(xgb, X, y, rounds, model=None):
    d = xgb.DMatrix(X, label=y)
    return xgb.train(dict(objective="survival:cox", max_depth=6, eta=0.3, subsample=0.8, seed=1), d, num_boost_round=rounds,
                     xgb_model=model, verbose_eval=False)


def test_cox_training_is_deterministic_and_resumes(xgb, tmp_path):
    X, y = _cox_data(2_000_000, 8, 11)
    a = _cox_train(xgb, X, y, 4).save_raw("ubj")
    b = _cox_train(xgb, X, y, 4).save_raw("ubj")
    assert a == b
    half = _cox_train(xgb, X, y, 2)
    path = str(tmp_path / "ckpt.ubj")
    half.save_model(path)
    resumed = _cox_train(xgb, X, y, 2, model=path)
    assert bytes(resumed.save_raw("ubj")) == bytes(a)


@pytest.fixture(scope="module")
def aft_model(xgb):
    X, lo, hi = _aft_data(5000, 6, 13)
    d = xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
    params = dict(objective="survival:aft", aft_loss_distribution="logistic", aft_loss_distribution_scale=1.7, max_depth=4, eta=0.4)
    return X, d, xgb.train(params, d, num_boost_round=5, verbose_eval=False)


def test_serving_and_model_io(xgb, aft_model, tmp_path):
    X, d, bst = aft_model
    margin = bst.predict(d, output_margin=True)
    np.testing.assert_allclose(bst.predict(d), np.exp(margin.astype(np.float64)), rtol=3e-7, atol=0)     # expf on the device
    contribs = bst.predict(d, pred_contribs=True)
    np.testing.assert_allclose(contribs.sum(axis=1), margin, rtol=0, atol=1e-5)
    want = bst.predict(d)
    for fmt in ("json", "ubj"):
        path = str(tmp_path / ("m." + fmt))
        bst.save_model(path)
        back = xgb.Booster(model_file=path)
        np.testing.assert_array_equal(_u32(back.predict(d)), _u32(want))
        cfg = json.loads(back.save_config())["learner"]["objective"]
        assert cfg["name"] == "survival:aft"
        assert cfg["aft_loss_param"]["aft_loss_distribution"] == "logistic"
        assert float(cfg["aft_loss_param"]["aft_loss_distribution_scale"]) == pytest.approx(1.7)
    doc = json.loads(bytes(bst.save_raw("json")))
    assert doc["learner"]["objective"]["aft_loss_param"]["aft_loss_distribution"] == "logistic"
    back = pickle.loads(pickle.dumps(bst))
    np.testing.assert_array_equal(_u32(back.predict(d)), _u32(want))
    assert json.loads(back.save_config())["learner"]["objective"] == json.loads(bst.save_config())["learner"]["objective"]
    X2, y2 = _cox_data(3000, 4, 2)
    cox = xgb.train(dict(objective="survival:cox"), xgb.DMatrix(X2, label=y2), num_boost_round=2, verbose_eval=False)
    assert json.loads(bytes(cox.save_raw("json")))["learner"]["objective"] == {"name": "survival:cox"}


def test_container_style_string_hyperparameters(xgb, tmp_path):
    X, y = _cox_data(4000, 5, 17)
    path = tmp_path / "train.csv"
    np.savetxt(path, np.column_stack([y, X]), delimiter=",", fmt="%.6g")
    d = xgb.DMatrix(str(path) + "?format=csv&label_column=0")
    res = {}
    bst = xgb.train({"objective": "survival:cox", "eval_metric": "cox-nloglik", "max_depth": "4", "eta": "0.3"}, d, num_boost_round=5,
                    evals=[(d, "train")], evals_result=res, verbose_eval=False)
    hist = res["train"]["cox-nloglik"]
    assert len(hist) == 5 and hist[-1] < hist[0]
    assert np.all(bst.predict(d) > 0)


@pytest.mark.parametrize("extra", [dict(booster="dart", rate_drop=0.3, seed=2), dict(num_parallel_tree=2, subsample=0.7, seed=2)])
def test_dart_and_forest_with_aft(xgb, extra):
    X, lo, hi = _aft_data(8000, 6, 19)
    d = xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
    bst = xgb.Booster(dict(objective="survival:aft", max_depth=4, **extra), [d])
    for r in range(4):
        bst.update(d, r)
    cache = _be().booster_cached_margin(bst.handle, d.handle, 1)[:, 0]
    np.testing.assert_allclose(bst.predict(d, output_margin=True), cache, rtol=0, atol=1e-6)


def test_errors(xgb):
    X, lo, hi = _aft_data(500, 3, 23)

    def fails(match, params, **kw):
        d = xgb.DMatrix(X, **kw)
        with pytest.raises(xgb.core.XGBoostError, match=match):
            xgb.train(params, d, num_boost_round=1, verbose_eval=False)

    fails("label_lower_bound and label_upper_bound", dict(objective="survival:aft"), label=np.ones(500, np.float32))
    bad = lo.copy(); bad[7] = hi[7] * 2 if np.isfinite(hi[7]) else -1.0
    bad_hi = hi.copy(); bad_hi[7] = 0.5 * max(lo[7], 1.0); bad_lo = lo.copy(); bad_lo[7] = max(lo[7], 1.0)
    fails("label_upper_bound must be >= label_lower_bound", dict(objective="survival:aft"), label_lower_bound=bad_lo, label_upper_bound=bad_hi)
    neg = lo.copy(); neg[3] = -1.0
    fails("label_lower_bound must be >= 0", dict(objective="survival:aft"), label_lower_bound=neg, label_upper_bound=hi)
    fails("aft_loss_distribution", dict(objective="survival:aft", aft_loss_distribution="weibull"), label_lower_bound=lo, label_upper_bound=hi)
    fails("aft_loss_distribution_scale", dict(objective="survival:aft", aft_loss_distribution_scale=0), label_lower_bound=lo, label_upper_bound=hi)


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks(xgb, tmp_path):
    """AFT on 2 ranks is the 1-GPU model bit for bit; Cox is rejected on 2 ranks."""
    import subprocess
    import sys
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29617", os.path.join(root, "tests", "helpers", "survival_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, lo, hi = _aft_data(40000, 10, 29)
    single = xgb.train(dict(objective="survival:aft", max_depth=5, eta=0.3), xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi),
                       num_boost_round=3, verbose_eval=False)
    m1, m2 = _be().booster_export_model(single.handle), _be().booster_export_model(xgb.Booster(model_file=out).handle)
    assert_same_structure(m2, m1)
    np.testing.assert_array_equal(_u32(m2["split_cond"]), _u32(m1["split_cond"]))
    with open(out + ".cox") as f:
        assert "survival:cox is not supported with more than one GPU" in f.read()
