"""Pre-JSON model files (SURVEY.md section 8(f) row 4: "legacy binary + pickle loaders", serve_utils.py:171-197).
The product's C++ reader (csrc/legacy_io.cc, reached through XGBoosterLoadModelFromBuffer / UnserializeFromBuffer and the
host-only XGB200LegacyModelToUBJ) against the oracle's independent numpy reader (oracle/legacy_model.py) on the reference's
own two fixtures; corrupt buffers must come back as errors; on the GPU the loaded models must predict what the oracle's
traversal of the same arrays predicts."""
import ctypes as C
import os
import pickle
import sys

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "legacy")
SAVED = os.path.join(GOLD, "saved_booster_xgboost-model")
PICKLED = os.path.join(GOLD, "pickled_model_xgboost-model")
ARRAYS = ["base_weights", "default_left", "left_children", "right_children", "loss_changes", "parents", "split_conditions", "split_indices", "split_type", "sum_hessian"]


@pytest.fixture(scope="module")
def lib():
    import sagemaker_xgboost_container_b200          # noqa: F401  (registers the hyphenated package directory)
    from sagemaker_xgboost_container_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return C.CDLL(backend.LIB_PATH)


def _convert(lib, buf):
    n, out = C.c_uint64(), C.c_char_p()
    lib.XGB200LegacyModelToUBJ.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_char_p)]
    rc = lib.XGB200LegacyModelToUBJ(buf, len(buf), C.byref(n), C.byref(out))
    if rc != 0:
        lib.XGBGetLastError.restype = C.c_char_p
        raise RuntimeError(lib.XGBGetLastError().decode())
    return C.string_at(out, n.value)


def _pickled_handle():
    import types

    class _B:
        def __setstate__(self, s):
            self.state = s
    saved = {k: sys.modules.get(k) for k in ("xgboost", "xgboost.core")}
    m, c = types.ModuleType("xgboost"), types.ModuleType("xgboost.core")
    c.Booster = _B
    m.core = c
    sys.modules["xgboost"], sys.modules["xgboost.core"] = m, c
    try:
        with open(PICKLED, "rb") as f:
            return pickle.load(f).state
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _same_document(got, ref):
    gl, rl = got["learner"], ref["learner"]
    assert gl["objective"] == rl["objective"]
    assert {k: str(v) for k, v in gl["learner_model_param"].items() if k != "base_score"} == {k: v for k, v in rl["learner_model_param"].items() if k != "base_score"}
    assert float(gl["learner_model_param"]["base_score"]) == float(rl["learner_model_param"]["base_score"])
    assert dict(gl["attributes"]) == rl["attributes"]
    gm, rm = gl["gradient_booster"]["model"], rl["gradient_booster"]["model"]
    np.testing.assert_array_equal(np.asarray(gm["tree_info"]), rm["tree_info"])
    np.testing.assert_array_equal(np.asarray(gm["iteration_indptr"]), rm["iteration_indptr"])
    assert len(gm["trees"]) == len(rm["trees"]) == int(gm["gbtree_model_param"]["num_trees"])
    for tg, tr in zip(gm["trees"], rm["trees"]):
        assert tg["tree_param"] == tr["tree_param"]
        for k in ARRAYS:
            a, b = np.asarray(tg[k]), np.asarray(tr[k])
            assert a.shape == b.shape and a.tobytes() == b.astype(a.dtype).tobytes(), k      # floats compared by bit pattern
    assert list(got["version"]) == list(ref["version"])


def test_c_reader_matches_the_oracle_reader_on_the_reference_fixtures(lib):
    from oracle import legacy_model, ubjson
    raw = open(SAVED, "rb").read()
    ref = legacy_model.to_document(raw)
    assert ref["learner"]["objective"] == {"name": "multi:softprob", "softmax_multiclass_param": {"num_class": "3"}}     # what SURVEY 8(c).2 lists
    assert ref["learner"]["learner_model_param"]["num_feature"] == "4" and len(ref["learner"]["gradient_booster"]["model"]["trees"]) == 60
    _same_document(ubjson.loads(_convert(lib, raw)), ref)
    state = _pickled_handle()
    assert state["best_ntree_limit"] == 20 and state["feature_names"] == ["f0", "f1", "f2", "f3"]
    handle = bytes(state["handle"])
    assert legacy_model.model_section(handle) == raw                     # the pickle wraps the very same model bytes
    _same_document(ubjson.loads(_convert(lib, handle)), ref)


def test_c_reader_rejects_damaged_files_without_crashing(lib):
    raw = open(SAVED, "rb").read()
    rng = np.random.default_rng(3)
    for cut in [0, 3, 100, 136, 150, 170, 330, 480, 1000, len(raw) // 2, len(raw) - 80, len(raw) - 1]:
        with pytest.raises(RuntimeError):
            _convert(lib, raw[:cut])
    for _ in range(200):                                                 # flipped size fields must end in an error or a document, never a fault
        b = bytearray(raw)
        off = int(rng.integers(0, len(b) - 4))
        b[off:off + 4] = rng.integers(0, 256, 4, dtype=np.uint8).tobytes()
        try:
            _convert(lib, bytes(b))
        except RuntimeError:
            pass
    with pytest.raises(RuntimeError):
        _convert(lib, b'{"learner": {}}' + b" " * 200)                   # a JSON document is not a legacy model


def _iris_like(n=300, seed=5):
    rng = np.random.default_rng(seed)
    X = rng.uniform([4.0, 2.0, 1.0, 0.1], [8.0, 4.5, 7.0, 2.6], size=(n, 4)).astype(np.float32)
    X[rng.random((n, 4)) < 0.05] = np.nan
    return X


def _oracle_predictions(X):
    from oracle import gbt_oracle as O, legacy_model, ubjson
    m = ubjson.model_from_xgb_json(legacy_model.to_document(open(SAVED, "rb").read()))
    return m, O.predict_leaf(m, X)


def test_reference_loader_opens_both_fixtures_on_the_cpu_engine(monkeypatch, tmp_path):
    """serve_utils.get_loaded_booster's two branches (pickle.load, then Booster.load_model) through this package bound as
    `xgboost`, on the oracle-backed test engine"""
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    from oracle.engine import OracleBackend
    monkeypatch.setattr(backend, "_BACKEND", OracleBackend(error_cls=xgb.XGBoostError))
    xgb.install_as_xgboost()
    with open(PICKLED, "rb") as f:
        b1 = pickle.load(f)
    b2 = xgb.Booster()
    b2.load_model(SAVED)
    X = _iris_like()
    d = xgb.DMatrix(X)
    _, leaves = _oracle_predictions(X)
    for b in (b1, b2):
        assert b.num_features() == 4 and b.num_boosted_rounds() == 20
        assert "multi:softprob" in b.save_config()
        p = b.predict(d)
        assert p.shape == (len(X), 3) and np.allclose(p.sum(1), 1, atol=1e-5)
        np.testing.assert_array_equal(b.predict(d, pred_leaf=True).astype(np.int32), leaves)
    assert b1.feature_names == ["f0", "f1", "f2", "f3"] and b1.best_ntree_limit == 20 and b1.best_iteration == 19
    np.testing.assert_array_equal(b1.predict(d), b2.predict(d))
    p2 = tmp_path / "resaved"                                           # migrated: written back in the current format
    b2.save_model(str(p2))
    b3 = xgb.Booster(model_file=str(p2))
    np.testing.assert_array_equal(b3.predict(d), b2.predict(d))


@pytest.mark.gpu
def test_legacy_files_predict_like_the_oracle_on_the_device(xgb):
    """CUDA backend: Booster.load_model on the 1.0 binary file and pickle.load of the pickled Booster (the two things
    serve_utils.get_loaded_booster does), then serve_utils.predict's calls"""
    from oracle import gbt_oracle as O
    xgb.install_as_xgboost()
    X = _iris_like(5000)
    m, leaves = _oracle_predictions(X)
    d = xgb.DMatrix(X)
    b2 = xgb.Booster()
    b2.load_model(SAVED)
    with open(PICKLED, "rb") as f:
        b1 = pickle.load(f)
    margins = O.predict_margin(m, X)
    for b in (b1, b2):
        assert b.num_features() == 4 and b.num_boosted_rounds() == 20
        np.testing.assert_array_equal(b.predict(d, pred_leaf=True).astype(np.int32), leaves)
        p = b.predict(d, iteration_range=(0, 20), validate_features=False)      # serve_utils.py:244-250 with best_ntree_limit = 20
        assert p.shape == (len(X), 3) and np.allclose(p.sum(1), 1, atol=1e-5)
        np.testing.assert_array_equal(b.predict(d, output_margin=True).view(np.uint32), margins.view(np.uint32))   # same arrays, same fp32 sums
    np.testing.assert_array_equal(b1.predict(d), b2.predict(d))
    raw = b2.save_raw("ubj")                                            # round trip through the current format keeps the predictions
    b3 = xgb.Booster(model_file=raw)
    np.testing.assert_array_equal(b3.predict(d), b2.predict(d))


def test_pickles_in_upstreams_current_state_layout_open_too(monkeypatch):
    """xgboost >= 1.x pickles a Booster as its __dict__ with the serialized learner under "handle" (today UBJSON {Model, Config});
    a pickle written by the real package therefore reaches Booster.__setstate__ with that key and no "_raw"."""
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    from oracle.engine import OracleBackend
    monkeypatch.setattr(backend, "_BACKEND", OracleBackend(error_cls=xgb.XGBoostError))
    rng = np.random.default_rng(0)
    X = rng.standard_normal((200, 5)).astype(np.float32)
    y = (X[:, 0] > 0).astype(np.float32)
    d = xgb.DMatrix(X, label=y, feature_names=["a", "b", "c", "d", "e"])
    bst = xgb.train({"objective": "binary:logistic", "max_depth": 3}, d, num_boost_round=4, verbose_eval=False)
    own = bst.__getstate__()
    upstream_style = {"handle": bytearray(own["_raw"]), "feature_names": ["a", "b", "c", "d", "e"], "feature_types": None, "best_iteration": 3}
    b2 = xgb.Booster.__new__(xgb.Booster)
    b2.__setstate__(upstream_style)
    np.testing.assert_array_equal(b2.predict(d), bst.predict(d))
    assert b2.feature_names == ["a", "b", "c", "d", "e"] and b2.best_iteration == 3
    b3 = pickle.loads(pickle.dumps(b2))                                  # and our own layout still round-trips
    np.testing.assert_array_equal(b3.predict(d), bst.predict(d))
