"""Custom objectives on the GPU (run with `pytest -m gpu` on an H100): `train(obj=)`, `Booster.update(fobj)` and `Booster.boost`.
An objective that hands back the pairs the engine itself computes at the margin it was given (through a twin booster's
XGB200BoosterComputeGradient) trains the model of the built-in objective byte for byte; the margin it is handed is
predict(output_margin=True); hand-written losses, input layouts, errors, sklearn, cv and two ranks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from util import assert_same_structure, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
BASE = dict(tree_method="hist", max_bin=256, max_depth=5, eta=0.3, base_score=0.4)


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def twin_objective(xgb, params, first_round=0):
    """obj(margin, d): the configured objective's pairs at `margin`, without row sampling, from a twin booster; the round
    number is passed on for the objectives that draw per round (rank:ndcg's pairs)."""
    tp = dict(params, subsample=1.0, sampling_method="uniform")
    twin = xgb.Booster(tp)
    state = {"round": first_round}

    def obj(margin, d):
        gp = _be().booster_compute_gradient(twin.handle, d.handle, margin, round=state["round"])
        state["round"] += 1
        return gp[..., 0], gp[..., 1]
    return obj


def _ranking_data(n, F, seed):
    X, y = synth(n, F, seed, "reg")
    rel = np.clip(np.round(y * 2 + 2), 0, 4).astype(f32)
    sizes = np.full(n // 20, 20)
    return X, rel, sizes


def _case(xgb, name, n=6000, F=12):
    """(params, DMatrix) of one identity case."""
    p = dict(BASE)
    if name == "squarederror":
        X, y = synth(n, F, 1, "reg")
        return dict(p, objective="reg:squarederror"), xgb.DMatrix(X, label=y)
    if name == "weighted":
        X, y = synth(n, F, 2, "reg")
        w = np.random.default_rng(2).uniform(0.5, 2.0, n).astype(f32)
        return dict(p, objective="reg:squarederror"), xgb.DMatrix(X, label=y, weight=w)
    if name == "logistic-spw":
        X, y = synth(n, F, 3, "bin")
        return dict(p, objective="binary:logistic", scale_pos_weight=3.0), xgb.DMatrix(X, label=y)
    if name == "softprob":
        X, y = synth(n, F, 4, "multi", K=3)
        return dict(p, objective="multi:softprob", num_class=3, base_score=0.5), xgb.DMatrix(X, label=y)
    if name == "multi-target":
        X, y = synth(n, F, 5, "reg")
        Y = np.stack([y, -y, 0.5 * y + 0.1], axis=1).astype(f32)
        return dict(p, objective="reg:squarederror"), xgb.DMatrix(X, label=Y)
    if name == "ndcg":
        X, rel, sizes = _ranking_data(n, F, 6)
        d = xgb.DMatrix(X, label=rel)
        d.set_group(sizes)
        return dict(p, objective="rank:ndcg", base_score=0.5), d
    if name == "aft":
        X, y = synth(n, F, 7, "pos")
        lo = y.copy()
        hi = np.where(np.arange(n) % 3 == 0, np.inf, y * 1.5).astype(f32)
        return dict(p, objective="survival:aft", base_score=1.0), xgb.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
    if name == "cox":
        X, y = synth(n, F, 8, "pos")
        y = np.where(np.arange(n) % 4 == 0, -y, y).astype(f32)
        return dict(p, objective="survival:cox", base_score=1.0), xgb.DMatrix(X, label=y)
    if name == "poisson":
        X, y = synth(n, F, 9, "count")
        return dict(p, objective="count:poisson", base_score=1.0), xgb.DMatrix(X, label=y)
    X, y = synth(n, F, 10, "reg")
    d = xgb.DMatrix(X, label=y)
    q = dict(p, objective="reg:squarederror", seed=3)
    if name == "subsample":
        return dict(q, subsample=0.7), d
    if name == "colsample-bynode":
        return dict(q, colsample_bynode=0.5), d
    if name == "forest-subsample":
        return dict(q, num_parallel_tree=3, subsample=0.8), d
    if name == "gradient-based":
        return dict(q, sampling_method="gradient_based", subsample=0.5), d
    if name == "lossguide":
        return dict(q, grow_policy="lossguide", max_leaves=24, max_depth=0), d
    if name == "quantile-dmatrix":
        return q, xgb.QuantileDMatrix(X, label=y)
    raise KeyError(name)


CASES = ["squarederror", "weighted", "logistic-spw", "softprob", "multi-target", "ndcg", "aft", "cox", "poisson", "subsample",
         "colsample-bynode", "forest-subsample", "gradient-based", "lossguide", "quantile-dmatrix"]


@pytest.mark.parametrize("name", CASES)
def test_identity(xgb, name):
    """The engine's own pairs handed back through obj= train the built-in model, byte for byte after every round."""
    params, d = _case(xgb, name)
    obj = twin_objective(xgb, params)
    b1, b2 = xgb.Booster(params, [d]), xgb.Booster(params, [d])
    for i in range(4):
        b1.update(d, i)
        b2.update(d, i, obj)
        assert b2.num_boosted_rounds() == i + 1
        assert b1.save_raw("ubj") == b2.save_raw("ubj"), "round %d" % i


def test_identity_resumed(xgb):
    params, d = _case(xgb, "squarederror")
    start = xgb.train(params, d, num_boost_round=2, verbose_eval=False)
    built = xgb.train(params, d, num_boost_round=3, xgb_model=start, verbose_eval=False)
    custom = xgb.train(params, d, num_boost_round=3, xgb_model=start, obj=twin_objective(xgb, params, 2), verbose_eval=False)
    assert built.save_raw("ubj") == custom.save_raw("ubj")


@pytest.mark.parametrize("name,shape", [("squarederror", (6000,)), ("softprob", (6000, 3))])
def test_margin_is_predict_margin(xgb, name, shape):
    params, d = _case(xgb, name)
    seen = []
    bst = xgb.Booster(params, [d])
    inner = twin_objective(xgb, params)

    def obj(margin, dm):
        ref = bst.predict(dm, output_margin=True)
        assert margin.shape == shape == ref.shape
        assert margin.dtype == np.float32
        np.testing.assert_array_equal(margin.view(np.uint32), ref.view(np.uint32))
        seen.append(1)
        return inner(margin, dm)
    for i in range(4):
        bst.update(d, i, obj)
    assert len(seen) == 4


def _sq_obj(margin, d):
    y = d.get_label()
    return (margin - y).astype(f32), np.ones_like(margin, f32)


def test_handwritten_squared_error(xgb):
    params, d = _case(xgb, "squarederror")
    built = xgb.train(params, d, num_boost_round=5, verbose_eval=False)
    custom = xgb.train(params, d, num_boost_round=5, obj=_sq_obj, verbose_eval=False)
    assert built.save_raw("ubj") == custom.save_raw("ubj")


def test_handwritten_pseudo_huber_against_oracle(xgb):
    """Non-constant hessians: a numpy pseudo-Huber loss against the oracle grown from the same loss's pairs (PairTrainer) on
    the device grid."""
    import custom_objective_reference as CR
    n, F, slope = 20000, 16, 1.0
    X, y = synth(n, F, 11, "reg")
    params = dict(BASE, objective="reg:squarederror", base_score=0.25)

    def huber(margin, d):
        z = (margin - d.get_label()).astype(f32)
        s = f32(1) + (z / f32(slope)) ** 2
        r = np.sqrt(s).astype(f32)
        return (z / r).astype(f32), (f32(slope * slope) / (s * r)).astype(f32)
    bst = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=3, obj=huber, verbose_eval=False)
    t = CR.PairTrainer(params, X, params["base_score"])
    t.set_device_grid()
    dref = xgb.DMatrix(X, label=y)
    for _ in range(3):
        gr, he = huber(t.margins()[:, 0], dref)
        t.boost(gr, he)
    m_gpu, m_ref = _be().booster_export_model(bst.handle), t.model()
    assert_same_structure(m_gpu, m_ref)
    leaf = m_ref["left"] == -1
    assert float(np.abs(m_gpu["split_cond"][leaf] - m_ref["split_cond"][leaf]).max()) <= 1e-5


def test_base_score_not_estimated(xgb):
    X, y = synth(3000, 8, 12, "reg")
    y = y + 5.0
    bst = xgb.train(dict(objective="reg:squarederror", max_depth=3), xgb.DMatrix(X, label=y), num_boost_round=2, obj=_sq_obj, verbose_eval=False)
    cfg = json.loads(bst.save_config())
    assert float(cfg["learner"]["learner_model_param"]["base_score"]) == 0.5


def _reference_bytes(xgb, params, d, grad, hess):
    b = xgb.Booster(params, [d])
    b.boost(d, 0, np.ascontiguousarray(grad, f32), np.ascontiguousarray(hess, f32))
    return b.save_raw("ubj")


def _pairs(n, K, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, K)).astype(f32), rng.uniform(0.5, 2.0, (n, K)).astype(f32)


@pytest.mark.parametrize("K", [1, 3])
def test_host_inputs(xgb, K):
    params, d = _case(xgb, "softprob" if K == 3 else "squarederror")
    n = d.num_row()
    g, h = _pairs(n, K)
    ref = _reference_bytes(xgb, params, d, g, h)
    wide_g = np.zeros((n, 2 * K), np.float64)
    wide_g[:, ::2] = g
    wide_h = np.zeros((n, 2 * K), f32)
    wide_h[:, ::2] = h
    for gg, hh in ((g.astype(np.float64), h.astype(np.float64)), (wide_g[:, ::2], wide_h[:, ::2]), (g.reshape(-1), h.reshape(-1))):
        b = xgb.Booster(params, [d])
        b.boost(d, 0, gg, hh)
        assert b.save_raw("ubj") == ref


@pytest.mark.parametrize("K", [1, 3])
def test_device_inputs(xgb, K):
    import torch
    params, d = _case(xgb, "softprob" if K == 3 else "squarederror")
    n = d.num_row()
    g, h = _pairs(n, K, 1)
    ref = _reference_bytes(xgb, params, d, g, h)
    tg, th = torch.from_numpy(g).cuda(), torch.from_numpy(h).cuda()
    wide = torch.zeros((n, 2 * K), dtype=torch.float64, device="cuda")
    wide[:, 1::2] = tg.double()
    cases = [(tg, th), (tg.double(), th.double()), (wide[:, 1::2], th), (tg.reshape(-1), th.reshape(-1)), (tg.t().contiguous().t(), th)]
    for gg, hh in cases:
        b = xgb.Booster(params, [d])
        b.boost(d, 0, gg, hh)
        assert b.save_raw("ubj") == ref


class _Interface:
    """A CUDA array known only by its __cuda_array_interface__: v3 with the producer's stream (as cupy exports it), or v2
    without one."""

    def __init__(self, t, stream=None):
        self._t = t
        iface = dict(t.__cuda_array_interface__)
        if stream is not None:
            iface.update(version=3, stream=stream)
        self.__cuda_array_interface__ = iface


@pytest.mark.parametrize("kind", ["torch", "v3-stream", "no-stream"])
def test_device_inputs_ordered_after_producer(xgb, kind):
    """Gradients written on a non-default stream just before boost(), with no synchronisation by the caller: the engine
    reads them after the writes (torch: its current stream; v3: the named stream; no stream: a device synchronise)."""
    import torch
    params, d = _case(xgb, "squarederror")
    n = d.num_row()
    g0, h0 = _pairs(n, 1, 3)
    g1, h1 = _pairs(n, 1, 4)
    ref = xgb.Booster(params, [d])
    ref.boost(d, 0, g0, h0)
    ref.boost(d, 1, g1, h1)
    tg, th = torch.from_numpy(g1).cuda(), torch.from_numpy(h1).cuda()
    sg, sh = torch.empty_like(tg), torch.empty_like(th)
    big = torch.ones((1 << 26,), device="cuda")
    s = torch.cuda.Stream()
    b = xgb.Booster(params, [d])
    b.boost(d, 0, g0, h0)              # every buffer of the round exists now: the next round allocates and frees nothing
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        sg.fill_(float("nan"))
        sh.fill_(float("nan"))
        for _ in range(50):             # tens of milliseconds of work ahead of the writes
            big.mul_(1.0001)
        sg.copy_(tg)
        sh.copy_(th)
        if kind == "torch":
            b.boost(d, 1, sg, sh)
        elif kind == "v3-stream":
            b.boost(d, 1, _Interface(sg, s.cuda_stream), _Interface(sh, s.cuda_stream))
        else:
            b.boost(d, 1, _Interface(sg), _Interface(sh))
    assert b.save_raw("ubj") == ref.save_raw("ubj")


def _assert_raises_and_recovers(xgb, bst, d, fn, match):
    before = bst.num_boosted_rounds()
    with pytest.raises((xgb.XGBoostError, ValueError), match=match):
        fn()
    assert bst.num_boosted_rounds() == before
    bst.update(d, before, _sq_obj)
    assert bst.num_boosted_rounds() == before + 1


def test_errors(xgb):
    params, d = _case(xgb, "squarederror")
    n = d.num_row()
    bst = xgb.Booster(params, [d])
    g, h = _pairs(n, 1, 2)
    for bad_row, gv, hv, what in ((17, np.nan, 1.0, "not finite"), (4000, 1.0, np.inf, "not finite"), (123, 1.0, -0.5, "negative")):
        gg, hh = g.copy(), h.copy()
        gg[bad_row], hh[bad_row] = gv, hv
        gg[bad_row + 5] = np.nan                     # a later row: the smallest one is named
        _assert_raises_and_recovers(xgb, bst, d, lambda: bst.boost(d, 0, gg, hh), "row %d, output column 0.*%s" % (bad_row, what))
    _assert_raises_and_recovers(xgb, bst, d, lambda: bst.boost(d, 0, g[:-1], h[:-1]), r"shape \(5999, 1\)")
    _assert_raises_and_recovers(xgb, bst, d, lambda: bst.boost(d, 0, np.zeros((n, 3), f32), np.ones((n, 3), f32)), "multi:softprob")
    _assert_raises_and_recovers(xgb, bst, d, lambda: bst.boost(d, 0, g, h[:, :0]), "mismatch")
    _assert_raises_and_recovers(xgb, bst, d, lambda: bst.boost(d, 0, g.reshape(-1)[:-1], h.reshape(-1)[:-1]), "multiple")


@pytest.mark.parametrize("extra,match", [(dict(booster="dart"), "booster=dart"), (dict(objective="reg:absoluteerror"), "reg:absoluteerror"),
                                         (dict(objective="reg:quantileerror", quantile_alpha=0.5), "reg:quantileerror")])
def test_rejected_configurations(xgb, extra, match):
    params, d = _case(xgb, "squarederror")
    bst = xgb.Booster(dict(params, **extra), [d])
    with pytest.raises(xgb.XGBoostError, match=match):
        bst.update(d, 0, _sq_obj)
    assert bst.num_boosted_rounds() == 0


def test_rejected_process_type_update(xgb):
    params, d = _case(xgb, "squarederror")
    start = xgb.train(params, d, num_boost_round=2, verbose_eval=False)
    bst = xgb.Booster(dict(params, process_type="update", updater="refresh"), [d], model_file=start)
    with pytest.raises(xgb.XGBoostError, match="process_type=update"):
        bst.update(d, 0, _sq_obj)


def test_sklearn(xgb):
    X, y = synth(4000, 10, 13, "reg")

    def sq(y_true, y_pred):
        return (y_pred - y_true).astype(f32), np.ones_like(y_pred, f32)
    reg = xgb.XGBRegressor(objective=sq, n_estimators=4, max_depth=4, base_score=0.3).fit(X, y)
    ref = xgb.train(dict(objective="reg:squarederror", max_depth=4, base_score=0.3), xgb.DMatrix(X, label=y), num_boost_round=4, obj=_sq_obj,
                    verbose_eval=False)
    assert reg.get_booster().save_raw("ubj") == ref.save_raw("ubj")

    def logistic(y_true, y_pred):
        p = 1.0 / (1.0 + np.exp(-y_pred))
        return (p - y_true).astype(f32), np.maximum(p * (1 - p), 1e-16).astype(f32)
    Xb, yb = synth(4000, 10, 14, "bin")
    clf = xgb.XGBClassifier(objective=logistic, n_estimators=4, max_depth=4).fit(Xb, yb)
    pb = clf.predict_proba(Xb)
    assert pb.shape == (4000, 2)
    m = clf.get_booster().predict(xgb.DMatrix(Xb), output_margin=True)
    np.testing.assert_allclose(pb[:, 1], 1.0 / (1.0 + np.exp(-m)), rtol=1e-5)
    np.testing.assert_array_equal(clf.predict(Xb), np.argmax(pb, axis=1))

    def softmax(y_true, y_pred):
        e = np.exp(y_pred - y_pred.max(axis=1, keepdims=True))
        p = e / e.sum(axis=1, keepdims=True)
        onehot = np.eye(y_pred.shape[1], dtype=f32)[y_true.astype(int)]
        return (p - onehot).astype(f32), np.maximum(2 * p * (1 - p), 1e-16).astype(f32)
    Xm, ym = synth(4000, 10, 15, "multi", K=3)
    clf3 = xgb.XGBClassifier(objective=softmax, n_estimators=4, max_depth=4).fit(Xm, ym)
    pm = clf3.predict_proba(Xm)
    assert pm.shape == (4000, 3)
    np.testing.assert_allclose(pm.sum(axis=1), 1.0, rtol=1e-5)
    np.testing.assert_array_equal(clf3.predict(Xm), np.argmax(pm, axis=1))
    with pytest.raises(ValueError, match="not supported by XGBRanker"):
        xgb.XGBRanker(objective=sq).fit(X, y, group=[2000, 2000])


def test_cv_and_custom_metric(xgb):
    params, d = _case(xgb, "squarederror")
    res = xgb.cv(params, d, num_boost_round=3, nfold=3, obj=_sq_obj, metrics="rmse", as_pandas=False, shuffle=False)
    ref = xgb.cv(params, d, num_boost_round=3, nfold=3, metrics="rmse", as_pandas=False, shuffle=False)
    # the engine's metric sums are double atomics: fold values agree to their last bits
    assert res.keys() == ref.keys()
    for k in res:
        assert res[k] == pytest.approx(ref[k], rel=1e-12, abs=1e-15)
    seen = []

    def metric(pred, dm):
        seen.append(pred)
        return "mine", 0.0
    params, d = _case(xgb, "logistic-spw")
    bst = xgb.train(params, d, num_boost_round=2, obj=_sq_obj, evals=[(d, "train")], custom_metric=metric, verbose_eval=False)
    margin = bst.predict(d, output_margin=True)
    np.testing.assert_array_equal(seen[-1], margin)


def test_two_ranks(xgb, tmp_path):
    """Each rank passes its own shard's gradients: the 2-GPU model equals the 1-GPU model byte for byte."""
    try:
        import torch
        ngpu = torch.cuda.device_count()
    except Exception:
        ngpu = 0
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    n, F, rounds = 40000, 20, 4
    out = str(tmp_path / "model.ubj")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29641", os.path.join(ROOT, "tests", "helpers", "custom_objective_shard_worker.py"), out, str(n), str(F), str(rounds)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    X, y = synth(n, F, 21, "reg")
    single = xgb.train(dict(objective="reg:squarederror", max_depth=5, base_score=0.5), xgb.DMatrix(X, label=y), num_boost_round=rounds, obj=_sq_obj,
                       verbose_eval=False)
    assert xgb.Booster(model_file=out).save_raw("ubj") == single.save_raw("ubj")
