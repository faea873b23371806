"""Custom objectives on the CPU: the oracle's growth from caller-given pairs (tests/custom_objective_reference.py PairTrainer)
fed the oracle objective's own pairs reproduces the oracle's training; and the Python layer on the oracle engine: margins
handed to `obj` in predict's shape, a loss with non-constant hessians, the gradient layouts `boost` accepts, the sklearn
decorator, `cv(obj=)` and the errors."""
import numpy as np
import pytest

import custom_objective_reference as CR
from util import synth

f32 = np.float32
PARAMS = dict(objective="reg:squarederror", max_depth=3, eta=0.3, base_score=0.5)


@pytest.fixture
def xgb(monkeypatch):
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    monkeypatch.setattr(backend, "_BACKEND", CR.CustomObjectiveOracleBackend(error_cls=xgb.XGBoostError))
    return xgb


def _data(n=500, F=6):
    return synth(n, F, 3, "reg")


def _sq(margin, d):
    return (margin - d.get_label()).astype(f32), np.ones_like(margin, f32)


def _same_trees(a, b, exact=True):
    for k in ("tree_offset", "tree_info", "left", "right", "split_index", "default_left"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    for k in ("split_cond", "base_weight", "sum_hess"):
        if exact:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
        else:
            np.testing.assert_allclose(a[k], b[k], rtol=0, atol=1e-5, err_msg=k)


@pytest.mark.parametrize("name", ["squarederror", "weighted-pow2", "subsample-colsample", "logistic-device-grid"])
def test_pair_trainer_reproduces_update(name):
    """PairTrainer fed orc_gradient's pairs at its own margins grows the oracle trainer's trees: bit for bit where the pairs
    are carried exactly (unit or power-of-two hessians), within the parity bar on the device grid otherwise."""
    from oracle import gbt_oracle as O
    X, y = _data(2000, 8)
    params = dict(PARAMS, max_depth=4)
    w = None
    if name == "weighted-pow2":
        w = (2.0 ** np.random.default_rng(5).integers(-2, 3, 2000)).astype(f32)
    elif name == "subsample-colsample":
        params.update(subsample=0.7, colsample_bynode=0.5, seed=4)
    elif name == "logistic-device-grid":
        y = (y > 0).astype(f32)
        params.update(objective="binary:logistic")
    ref = O.Trainer(params, X=X, y=y, weights=w)
    pt = CR.PairTrainer(params, X, params["base_score"])
    if name == "logistic-device-grid":
        ref.set_device_grid()
        pt.set_device_grid()
    np.testing.assert_array_equal(pt.margins(), ref.margins())
    for _ in range(3):
        gp = O.gradient(params, pt.margins(), y, w)
        pt.boost(gp[:, 0, 0], gp[:, 0, 1])
        ref.update()
    _same_trees(pt.model(), ref.model(), exact=name != "logistic-device-grid")
    np.testing.assert_allclose(pt.margins(), ref.margins(), rtol=0, atol=1e-5 if name == "logistic-device-grid" else 0)


def test_carrier_within_one_ulp():
    """The carried g is g itself where a float32 label gives it, and within one ulp of g everywhere; h is carried exactly."""
    rng = np.random.default_rng(9)
    g, h = rng.standard_normal(100000).astype(f32), rng.uniform(0.01, 3.0, 100000).astype(f32)
    carried = (-CR.carrier(g, h) * h).astype(f32)
    assert np.all(np.abs(carried - g) <= np.spacing(np.abs(g)))
    assert np.array_equal((-CR.carrier(g, np.ones_like(h)) * f32(1)).astype(f32), g)
    with pytest.raises(ValueError):
        CR.carrier(np.ones(2, f32), np.zeros(2, f32))


def test_pseudo_huber_obj(xgb):
    """A loss with non-constant hessians through obj= against the oracle's reg:pseudohubererror, at the parity bar."""
    from oracle import gbt_oracle as O
    X, y = _data()

    def huber(margin, d):
        z = (margin - d.get_label()).astype(f32)
        s = f32(1) + z * z
        r = np.sqrt(s).astype(f32)
        return (z / r).astype(f32), (f32(1) / (s * r)).astype(f32)
    bst = xgb.train(PARAMS, xgb.DMatrix(X, label=y), num_boost_round=3, obj=huber, verbose_eval=False)
    ref = O.train(dict(PARAMS, objective="reg:pseudohubererror", huber_slope=1.0), X, y, 3).model()
    _same_trees(bst.handle.model(), ref, exact=False)


def test_train_obj_equals_builtin(xgb):
    X, y = _data()
    d = xgb.DMatrix(X, label=y)
    seen = []

    def obj(margin, dm):
        seen.append(margin.copy())
        return _sq(margin, dm)
    custom = xgb.train(PARAMS, d, num_boost_round=3, obj=obj, verbose_eval=False)
    built = xgb.train(PARAMS, d, num_boost_round=3, verbose_eval=False)
    assert custom.save_raw("json") == built.save_raw("json")
    assert [m.shape for m in seen] == [(500,)] * 3
    np.testing.assert_array_equal(seen[0], np.full(500, 0.5, f32))


@pytest.mark.parametrize("layout", ["float64", "strided", "flat", "int"])
def test_boost_layouts(xgb, layout):
    X, y = _data()
    d = xgb.DMatrix(X, label=y)
    ref = xgb.Booster(PARAMS, [d])
    ref.update(d, 0)
    bst = xgb.Booster(PARAMS, [d])
    g, h = _sq(np.full(500, 0.5, f32), d)
    if layout == "float64":
        g, h = g.astype(np.float64), h.astype(np.float64)
    elif layout == "strided":
        wide = np.zeros((500, 2), f32)
        wide[:, 1] = g
        g = wide[:, 1:]
    elif layout == "flat":
        g, h = g.reshape(-1), h.reshape(-1)
    else:                                    # other dtypes go to float32 on the host
        h = np.ones(500, np.int32)
    bst.boost(d, 0, g, h)
    assert bst.save_raw("json") == ref.save_raw("json")


def test_boost_errors(xgb):
    X, y = _data()
    d = xgb.DMatrix(X, label=y)
    bst = xgb.Booster(PARAMS, [d])
    g, h = _sq(np.full(500, 0.5, f32), d)
    bst.boost(d, 0, g, h)
    g, h = _sq(bst.predict(d, output_margin=True), d)
    with pytest.raises(ValueError, match="not a multiple"):
        bst.boost(d, 0, g[:-1], h[:-1])
    with pytest.raises(ValueError, match="mismatch"):
        bst.boost(d, 0, g, np.ones((500, 2), f32))
    with pytest.raises(ValueError, match="1- or 2-dimensional"):
        bst.boost(d, 0, g.reshape(500, 1, 1), h.reshape(500, 1, 1))
    with pytest.raises(xgb.XGBoostError, match="shape"):
        bst.boost(d, 0, np.zeros((500, 2), f32), np.ones((500, 2), f32))
    bad = h.copy()
    bad[7] = -1
    with pytest.raises(xgb.XGBoostError, match="row 7"):
        bst.boost(d, 0, g, bad)
    assert bst.num_boosted_rounds() == 1
    bst.boost(d, 1, g, h)
    assert bst.num_boosted_rounds() == 2
    with pytest.raises(TypeError):
        bst.boost(X, 0, g, h)


def test_sklearn_decorator(xgb):
    X, y = _data()

    def sq(y_true, y_pred):
        assert y_true.shape == y_pred.shape == (500,)
        return (y_pred - y_true).astype(f32), np.ones_like(y_pred, f32)
    reg = xgb.XGBRegressor(objective=sq, n_estimators=3, max_depth=3, base_score=0.5).fit(X, y)
    ref = xgb.train(PARAMS, xgb.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    assert reg.get_booster().save_raw("json") == ref.save_raw("json")
    assert reg.get_xgb_params()["objective"] == "reg:squarederror"
    with pytest.raises(ValueError, match="custom objective function not supported by XGBRanker"):
        xgb.XGBRanker(objective=sq).fit(X, y, group=[250, 250])


def test_cv_obj(xgb):
    X, y = _data()
    d = xgb.DMatrix(X, label=y)
    res = xgb.cv(PARAMS, d, num_boost_round=2, nfold=2, obj=_sq, metrics="rmse", as_pandas=False, shuffle=False)
    ref = xgb.cv(PARAMS, d, num_boost_round=2, nfold=2, metrics="rmse", as_pandas=False, shuffle=False)
    assert res == ref
