"""In-place prediction without a GPU: the host half of csrc/inplace.h (typestr parsing, the row chunks of host inputs) over a
sweep compiled with g++ (tests/helpers/inplace_sweep.cc), and the Python layer of `Booster.inplace_predict` on the oracle
engine (tests/inplace_reference.py): each input kind, dtype and layout gives predict(DMatrix(Xf)), with the shapes, base
margins and errors of the CUDA engine."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from inplace_reference import InplaceOracleBackend
from util import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sagemaker-xgboost-container_b200", "csrc")


@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path_factory.mktemp("inplace") / "sweep")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-fsanitize=undefined", "-I", CSRC,
           os.path.join(ROOT, "tests", "helpers", "inplace_sweep.cc"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, UBSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0 and not r.stderr, (r.stdout + r.stderr)[-3000:]
    return json.loads(r.stdout)


def test_chunk_plans_cover_the_rows_within_the_cap(sweep):
    assert sweep["violations"] == 0
    assert sweep["dense_plans"] > 500 and sweep["csr_plans"] == 3000 and sweep["multi_chunk"] > 1000 and sweep["refused"] > 0


def test_typestrs(sweep):
    t = sweep["types"]
    assert [t[k][0] for k in ("<f4", "<f8", "<f2", "|i1", "<i2", "<i4", "<i8", "|u1", "<u2", "<u4", "<u8", "|b1")] == list(range(12))
    assert [t[k][1] for k in ("<f4", "<f8", "<f2", "|i1", "<i8", "|u1", "<u8", "|b1")] == [4, 8, 2, 1, 8, 1, 8, 1]
    for k, word in (("<c8", "complex"), ("<c16", "complex"), ("|O", "object"), ("<M8[ns]", "datetime"), ("<m8[s]", "timedelta"),
                    (">f4", "big-endian"), ("<V8", "unsupported")):
        assert t[k][0] == -1 and word in t[k][2], (k, t[k])


@pytest.fixture
def xgb(monkeypatch):
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    monkeypatch.setattr(backend, "_BACKEND", InplaceOracleBackend(error_cls=xgb.XGBoostError))
    return xgb


def _model(xgb, F=6, K=1, rounds=4):
    X, y = synth(400, F, 2, "multi" if K > 1 else "reg", K=K, quantised=False)
    params = dict(max_depth=3, eta=0.3, base_score=0.5)
    if K > 1:
        params.update(objective="multi:softprob", num_class=K)
    return xgb.train(params, xgb.DMatrix(X, label=y), rounds), X


def _same(a, b):
    assert type(a) is np.ndarray and a.dtype == np.float32 and a.shape == b.shape
    np.testing.assert_array_equal(a.view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("dtype", ["float32", "float64", "float16", "int8", "int32", "int64", "uint8", "uint64", "bool"])
@pytest.mark.parametrize("layout", ["C", "F", "rows", "cols", "reversed"])
def test_dense_dtypes_and_layouts(xgb, dtype, layout):
    bst, X = _model(xgb)
    A = (X * 3).astype(dtype) if dtype != "bool" else X > 0
    if layout == "F":
        A = np.asfortranarray(A)
    elif layout == "rows":
        A = A[::3]
    elif layout == "cols":
        A = np.ascontiguousarray(np.concatenate([A, A], axis=1))[:, ::2]
    elif layout == "reversed":
        A = A[::-1, ::-1][:, ::-1]
    for missing in (np.nan, 0.0, -999.0):
        for ptype in ("value", "margin"):
            got = bst.inplace_predict(A, missing=missing, predict_type=ptype)
            want = bst.predict(xgb.DMatrix(np.asarray(A).astype(np.float32), missing=missing), output_margin=ptype == "margin")
            _same(got, want)


def test_csr_csc_pandas_and_shapes(xgb):
    import scipy.sparse as sp
    bst, X = _model(xgb, K=3)
    Xs = X.copy()
    Xs[np.random.default_rng(3).random(X.shape) < 0.5] = 0
    csr = sp.csr_matrix(Xs)
    want = bst.predict(xgb.DMatrix(csr))
    _same(bst.inplace_predict(csr), want)
    _same(bst.inplace_predict(csr.tocsc()), want)
    pd = pytest.importorskip("pandas")
    df = pd.DataFrame({"a%d" % j: X[:, j].astype(np.float64 if j % 2 else np.float32) for j in range(X.shape[1])})
    _same(bst.inplace_predict(df, validate_features=False), bst.predict(xgb.DMatrix(df), validate_features=False))
    assert bst.inplace_predict(X[:1]).shape == (1, 3)
    assert bst.inplace_predict(X[:0]).shape == (0, 3)
    assert bst.inplace_predict(X, predict_type="margin", strict_shape=True).shape == (400, 3)
    bm = np.random.default_rng(4).standard_normal((400, 3)).astype(np.float32)
    _same(bst.inplace_predict(X, base_margin=bm, predict_type="margin"),
          bst.predict(xgb.DMatrix(X, base_margin=bm.reshape(-1)), output_margin=True))


def test_one_column_and_strict_shape(xgb):
    bst, X = _model(xgb, F=1)
    _same(bst.inplace_predict(X[:, 0]), bst.predict(xgb.DMatrix(X)))
    assert bst.inplace_predict(X, strict_shape=True).shape == (400, 1)
    _same(bst.inplace_predict(X, iteration_range=(1, 3)), bst.predict(xgb.DMatrix(X), iteration_range=(1, 3)))


def test_errors(xgb):
    bst, X = _model(xgb)
    with pytest.raises(ValueError, match="predict_type"):
        bst.inplace_predict(X, predict_type="leaf")
    with pytest.raises(xgb.XGBoostError, match="2-dimensional"):
        bst.inplace_predict(X.reshape(400, 3, 2), validate_features=False)
    with pytest.raises(xgb.XGBoostError, match="typestr"):
        bst.inplace_predict(X.astype(np.complex64))
    with pytest.raises(xgb.XGBoostError, match="feature count"):
        bst.inplace_predict(np.concatenate([X, X], axis=1))
    with pytest.raises(xgb.XGBoostError, match="base_margin"):
        bst.inplace_predict(X, base_margin=np.zeros(3, np.float32))
    _same(bst.inplace_predict(X), bst.predict(xgb.DMatrix(X)))
