"""CPU checks of the booster=dart restatement (tests/dart_reference.py) and of the container route on the oracle engine with
booster=dart."""
import os
import re

import numpy as np
import pytest

import dart_reference as DR
import reference_stubs
from util import synth

f32 = np.float32


def _dp(**kw):
    return dict(dict(rate_drop=0.0, skip_drop=0.0, one_drop=0, sample_type="uniform", normalize_type="tree"), **kw)


@pytest.mark.parametrize("sample_type", ["uniform", "weighted"])
def test_skip_drop_one_never_drops(sample_type):
    w = [f32(1)] * 30
    for rnd in range(1, 40):
        assert DR.drop_set(w, rnd, 3, _dp(rate_drop=1.0, one_drop=1, skip_drop=1.0, sample_type=sample_type)) == []


@pytest.mark.parametrize("sample_type", ["uniform", "weighted"])
def test_rate_drop_one_drops_every_tree(sample_type):
    w = [f32(1)] * 12
    for rnd in range(1, 20):
        assert DR.drop_set(w, rnd, 5, _dp(rate_drop=1.0, sample_type=sample_type)) == list(range(12))


@pytest.mark.parametrize("sample_type", ["uniform", "weighted"])
def test_one_drop_always_drops_a_tree_after_round_zero(oracle, sample_type):
    X, y = synth(600, 5, 2, "reg")
    t = DR.DartTrainer(dict(objective="reg:squarederror", max_depth=3, eta=0.3, rate_drop=0.0, one_drop=1, sample_type=sample_type, seed=1), X, y)
    for _ in range(8):
        t.update()
    assert t.drops[0] == [] and all(len(D) == 1 for D in t.drops[1:])
    assert len(set(D[0] for D in t.drops[1:])) > 1


def test_normalisation_by_hand():
    # tree: dropped *= |D| / (|D| + lr), new = 1 / (|D| + lr); forest: both 1 / (1 + lr); lr = eta / K
    lr = f32(0.3 / 2)
    assert DR.normalisation(3, 0.3, 2, "tree") == (f32(3 / float(f32(3 + lr))), f32(1 / float(f32(3 + lr))))
    assert DR.normalisation(3, 0.3, 2, "forest") == (f32(1 / (1 + float(lr))), f32(1 / (1 + float(lr))))
    assert DR.normalisation(0, 0.3, 2, "tree") == (f32(1), f32(1))
    X, y = synth(800, 6, 4, "reg")
    for nt in ("tree", "forest"):
        t = DR.DartTrainer(dict(objective="reg:squarederror", max_depth=3, eta=0.5, rate_drop=0.5, normalize_type=nt, seed=2), X, y)
        w = []
        for _ in range(10):
            D = t.update()
            fac, new = DR.normalisation(len(D), 0.5, 1, nt)
            w = [f32(v * fac) if i in D else v for i, v in enumerate(w)] + [new]
            assert [float(v) for v in t.weights] == [float(v) for v in w]
        assert any(v != 1 for v in w)


def test_rate_drop_zero_is_the_plain_trainer(oracle):
    X, y = synth(1000, 6, 8, "reg")
    params = dict(objective="reg:squarederror", max_depth=4, eta=0.3, seed=1)
    t = DR.DartTrainer(dict(params, rate_drop=0.0), X, y)
    p = oracle.Trainer(params, X=X, y=y)
    for _ in range(5):
        t.update(); p.update()
    np.testing.assert_array_equal(t.m_full, p.margins())
    np.testing.assert_array_equal(DR.predict_margin(t.model(), X, t.weights), oracle.predict_margin(p.model(), X))


def test_parameters_reach_the_engine():
    from sagemaker_xgboost_container_b200 import core
    for k, v in (("rate_drop", 0.1), ("one_drop", 1), ("skip_drop", 0.5), ("sample_type", "weighted"), ("normalize_type", "forest")):
        assert core._check_unapplied(k, v) == v


@pytest.mark.skipif(not reference_stubs.reference_available(), reason="the reference container is not mounted here")
def test_sagemaker_train_with_dart_on_the_oracle_engine(monkeypatch, tmp_path, capsys):
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    monkeypatch.setattr(backend, "_BACKEND", DR.DartOracleBackend(error_cls=xgb.XGBoostError))
    reference_stubs.install(xgb)
    from sagemaker_xgboost_container.algorithm_mode import train as ref_train
    X, y = synth(1500, 6, 12, "reg")
    tr = tmp_path / "train"
    tr.mkdir()
    np.savetxt(tr / "train.csv", np.column_stack([y, X]), delimiter=",", fmt="%.6f")
    data_config = {"train": {"ContentType": "text/csv", "TrainingInputMode": "File", "S3DistributionType": "FullyReplicated"}}
    hp = {"objective": "reg:squarederror", "num_round": "12", "max_depth": "4", "eta": "0.3", "booster": "dart", "rate_drop": "0.3",
          "sample_type": "weighted", "normalize_type": "forest", "one_drop": "1", "skip_drop": "0.1"}
    model_dir = tmp_path / "model"
    ref_train.sagemaker_train(train_config=hp, data_config=data_config, train_path=str(tr), val_path=None, model_dir=str(model_dir),
                              sm_hosts=["algo-1"], sm_current_host="algo-1", checkpoint_config={})
    lines = [l for l in capsys.readouterr().out.splitlines() if re.match(r"^\[\d+\]\ttrain-rmse:", l)]
    assert len(lines) == 12
    from oracle import ubjson
    doc = ubjson.load(str(model_dir / "xgboost-model"))
    gb = doc["learner"]["gradient_booster"]
    assert gb["name"] == "dart" and len(gb["weight_drop"]) == 12 and any(float(v) != 1 for v in gb["weight_drop"])
    bad = dict(hp, sample_type="gaussian")
    with pytest.raises(Exception) as e:
        ref_train.sagemaker_train(train_config=bad, data_config=data_config, train_path=str(tr), val_path=None, model_dir=str(tmp_path / "m2"),
                                  sm_hosts=["algo-1"], sm_current_host="algo-1", checkpoint_config={})
    assert "sample_type" in str(e.value) or "UserError" in type(e.value).__name__ or isinstance(e.value, xgb.XGBoostError)
