"""`Booster.inplace_predict` on the GPU (run with `pytest -m gpu` on an H100).  Every assertion is a bit-equality against
predict(DMatrix(Xf)) on the same booster, Xf being the input converted to float32 as the DMatrix path converts it
(np.asarray(X).astype(np.float32), t.float().contiguous(), the CSR with float32 data): dtypes, layouts, host and CUDA inputs,
missing values, CSR and pandas inputs, every branch of the predictor's plan, every model kind, the chunked host path across
chunk boundaries, the errors, and the C entries called through ctypes with upstream's argument order."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import test_gpu_predict as P
from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = ["float32", "float64", "float16", "int8", "int32", "int64", "uint8", "uint64", "bool"]


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _host(a):
    return a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)


def _same(got, want):
    got = _host(got)
    assert got.dtype == np.float32 and got.shape == want.shape, (got.dtype, got.shape, want.shape)
    np.testing.assert_array_equal(got.view(np.uint32), np.ascontiguousarray(want, np.float32).view(np.uint32))


def _ref(xgb, bst, Xf, missing=np.nan, **kw):
    return bst.predict(xgb.DMatrix(np.asarray(Xf, np.float32), missing=missing), **kw)


def _cast(X, dtype, scale=3.0):
    """X in dtype: integers from scaled values (NaN -> 0), bool from the sign"""
    if dtype == "bool":
        return np.nan_to_num(X) > 0
    if dtype.startswith(("int", "uint")):
        Y = np.nan_to_num(X * scale)
        if dtype.startswith("uint"):
            Y = np.abs(Y)
        return Y.astype(dtype)
    return X.astype(dtype)


@pytest.fixture(scope="module")
def model(xgb):
    """20 rounds of depth 6 on 28 features with missing values; the predictor tiles it in one chunk"""
    X, y = synth(20000, 28, 3, "reg", quantised=False, missing_frac=0.1)
    bst = xgb.train(dict(tree_method="hist", max_depth=6, eta=0.3), xgb.DMatrix(X, label=y), 20)
    return bst, X


# ------------------------------------------------------------------------------------------------------ dtypes and layouts
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", ["host", "cuda"])
def test_dtypes(xgb, model, dtype, where):
    import torch
    bst, X = model
    A = _cast(X, dtype)
    want = _ref(xgb, bst, A.astype(np.float32))
    if where == "host":
        _same(bst.inplace_predict(A), want)
        return
    t = torch.from_numpy(np.ascontiguousarray(A)).cuda()
    got = bst.inplace_predict(t)
    assert isinstance(got, torch.Tensor) and got.is_cuda
    _same(got, _ref(xgb, bst, t.float().contiguous().cpu().numpy()))
    _same(got, want)


def test_float64_on_and_next_to_thresholds(xgb, model):
    """float64 values that round onto each split threshold (the threshold, +- one double ulp) and int64 above 2^24"""
    import torch
    bst, _ = model
    m = _be().booster_export_model(bst.handle)
    internal = m["left"] != -1
    f, cond = m["split_index"][internal], m["split_cond"][internal].astype(np.float64)
    cols = []
    for d in (-np.inf, 0, np.inf):
        v = cond if d == 0 else np.nextafter(cond, d)
        cols.append(v)
    vals = np.concatenate(cols)
    feats = np.concatenate([f, f, f])
    X = np.full((len(vals), 28), np.nan)
    X[np.arange(len(vals)), feats] = vals
    X[:, 0] = np.where(np.isnan(X[:, 0]), vals, X[:, 0])
    assert np.array_equal(X.astype(np.float32)[np.arange(len(vals)), feats], np.concatenate([cond, cond, cond]).astype(np.float32))
    want = _ref(xgb, bst, X.astype(np.float32))
    _same(bst.inplace_predict(X), want)
    _same(bst.inplace_predict(torch.from_numpy(X).cuda()), want)
    big = (np.arange(28 * 50, dtype=np.int64).reshape(50, 28) * 7919 + (1 << 24) + 1) * np.where(np.arange(28) % 2, 1, -1)
    big[0, :] = np.iinfo(np.int64).max
    _same(bst.inplace_predict(big), _ref(xgb, bst, big.astype(np.float32)))
    _same(bst.inplace_predict(torch.from_numpy(big).cuda()), _ref(xgb, bst, big.astype(np.float32)))
    u = (np.abs(big) * 3).astype(np.uint64)
    u[1, :] = np.iinfo(np.uint64).max
    _same(bst.inplace_predict(u), _ref(xgb, bst, u.astype(np.float32)))


def _layouts(X):
    W = np.concatenate([X, X[:, ::-1]], axis=1)
    return {"C": X, "F": np.asfortranarray(X), "row_slice": X[1000:9000:3], "col_slice": W[:, :28], "col_step": np.ascontiguousarray(np.repeat(X, 2, axis=1))[:, ::2],
            "negative": X[::-1], "negative_cols": np.ascontiguousarray(X[:, ::-1])[::-2, ::-1]}


@pytest.mark.parametrize("dtype", ["float32", "float64", "float16", "int32"])
def test_layouts_host_and_cuda(xgb, model, dtype):
    import torch
    bst, X = model
    for name, A in _layouts(_cast(X, dtype)).items():
        want = _ref(xgb, bst, np.asarray(A).astype(np.float32))
        _same(bst.inplace_predict(A), want)
        if name.startswith("negative"):
            continue                                       # torch has no negative strides
        t = torch.from_numpy(np.ascontiguousarray(A)).cuda()
        views = {"C": t, "F": t.t().contiguous().t(), "row_slice": torch.from_numpy(_cast(X, dtype)).cuda()[1000:9000:3],
                 "col_slice": torch.from_numpy(np.concatenate([_cast(X, dtype)] * 2, axis=1)).cuda()[:, :28],
                 "col_step": torch.from_numpy(np.ascontiguousarray(np.repeat(_cast(X, dtype), 2, axis=1))).cuda()[:, ::2]}
        v = views[name]
        _same(bst.inplace_predict(v), want)
    T = torch.from_numpy(np.ascontiguousarray(_cast(X, dtype).T)).cuda()          # (28, n) contiguous; .t() is (n, 28) F order
    _same(bst.inplace_predict(T.t()), _ref(xgb, bst, T.t().float().contiguous().cpu().numpy()))


def test_tensor_written_on_a_side_stream(xgb, model):
    import torch
    bst, X = model
    want = _ref(xgb, bst, X)
    src = torch.from_numpy(X).cuda()
    big = torch.randn(4096, 4096, device="cuda")
    side = torch.cuda.Stream()
    out = torch.empty_like(src)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(8):
            big = big @ big / 64.0                        # keeps the side stream busy before the write
        out.copy_(src + 0.0 * big[0, 0])
        got = bst.inplace_predict(out)                    # no synchronisation by the caller: the tensor's current stream is named
    torch.cuda.synchronize()
    _same(got, want)
    # a v3 interface with the stream, and one without any stream key (a device synchronise)
    for with_stream in (True, False):
        out2 = torch.empty_like(src)
        with torch.cuda.stream(side):
            out2.copy_(src + 0.0 * (big @ big)[0, 0])
            iface = dict(out2.__cuda_array_interface__)
            if with_stream:
                iface["stream"] = side.cuda_stream
            else:
                iface.pop("stream", None)
            holder = type("Iface", (), {})()
            holder.__cuda_array_interface__ = iface
            holder._keep = out2
            got = bst.inplace_predict(holder)
        torch.cuda.synchronize()
        _same(got, want)


# ------------------------------------------------------------------------------------------------------ missing values, CSR, pandas
@pytest.mark.parametrize("missing", [np.nan, 0.0, -999.0])
def test_missing(xgb, model, missing):
    import torch
    bst, X = model
    A = X.copy()
    A[::7, 3] = 0.0
    A[::5, 5] = -999.0
    A[::11, 7] = -0.0
    for dtype in ("float32", "float64", "int32"):
        B = _cast(A, dtype, 1.0) if dtype == "int32" else A.astype(dtype)
        want = _ref(xgb, bst, B.astype(np.float32), missing=missing)
        _same(bst.inplace_predict(B, missing=missing), want)
        _same(bst.inplace_predict(torch.from_numpy(B).cuda(), missing=missing), want)


def test_csr(xgb, model):
    import scipy.sparse as sp
    bst, X = model
    rng = np.random.default_rng(9)
    n, F = 3000, 28
    indptr = [0]
    indices, data = [], []
    for r in range(n):
        k = 0 if r % 10 == 0 else int(rng.integers(0, 40))            # empty rows, and rows longer than F (duplicates)
        cols = rng.integers(0, F, k)                                   # unsorted, repeated
        vals = rng.standard_normal(k)
        vals[rng.random(k) < 0.2] = 0.0                                # explicit zeros stay
        indices.extend(cols.tolist()); data.extend(vals.tolist()); indptr.append(len(indices))
    for dt in (np.float32, np.float64):
        csr = sp.csr_matrix((np.asarray(data, dt), np.asarray(indices, np.int32), np.asarray(indptr, np.int64)), shape=(n, F))
        csr32 = sp.csr_matrix((csr.data.astype(np.float32), csr.indices, csr.indptr), shape=(n, F))
        want = bst.predict(xgb.DMatrix(csr32))
        for missing in (np.nan, 0.0):
            _same(bst.inplace_predict(csr, missing=missing), want)
        try:
            _be().booster_inplace_debug(bst.handle, 17)                # several chunks
            _same(bst.inplace_predict(csr), want)
        finally:
            _be().booster_inplace_debug(bst.handle, 0)
    csc = sp.random(2000, F, density=0.3, random_state=1, format="csc", dtype=np.float32)
    _same(bst.inplace_predict(csc), bst.predict(xgb.DMatrix(csc.tocsr())))


def test_pandas(xgb, model):
    pd = pytest.importorskip("pandas")
    bst, X = model
    cols = {}
    for j in range(28):
        kind = j % 4
        v = X[:, j]
        cols["f%d" % j] = v.astype(np.float64) if kind == 0 else (np.nan_to_num(v * 5).astype(np.int64) if kind == 1 else
                                                                  (np.nan_to_num(v * 5).astype(np.int8) if kind == 2 else v))
    df = pd.DataFrame(cols)
    bst2 = bst.copy()
    _same(bst2.inplace_predict(df, validate_features=False), bst2.predict(xgb.DMatrix(df), validate_features=False))
    same = pd.DataFrame({"f%d" % j: X[:, j].astype(np.float64) for j in range(28)})
    _same(bst2.inplace_predict(same, validate_features=False, missing=0.5), bst2.predict(xgb.DMatrix(same, missing=0.5), validate_features=False))


# ------------------------------------------------------------------------------------------------------ predictor plans
def _check_plan(xgb, f, X, reason=None):
    import torch
    d = xgb.DMatrix(X)
    plan = f.plan(d)
    if reason is None:
        assert plan["kernel"] == P.TILED, plan
    else:
        assert plan["kernel"] == P.PER_ROW and plan["reason"] == reason, plan
    want = f.bst.predict(d, output_margin=True)
    _same(f.bst.inplace_predict(X, predict_type="margin"), want)
    _same(f.bst.inplace_predict(X.astype(np.float64), predict_type="margin"), want)
    _same(f.bst.inplace_predict(torch.from_numpy(np.asfortranarray(X).T.copy()).cuda().t(), predict_type="margin"), want)
    return plan


def test_plans(xgb):
    one = P._train(xgb, dict(max_depth=6), 20, 7)
    X, _ = synth(5000, 20, 11, "reg", quantised=False, missing_frac=0.1)
    assert len(_check_plan(xgb, one, X)["chunks"]) == 1
    several = P._train(xgb, dict(max_depth=6), 28, 100, n=30000, seed=6, slots=True)
    X28, _ = synth(5000, 28, 12, "reg", quantised=False, missing_frac=0.1)
    assert len(_check_plan(xgb, several, X28)["chunks"]) > 1
    wide = P._train(xgb, dict(max_depth=6), 1300, 10, n=3000, seed=8)
    Xw, _ = synth(700, 1300, 13, "reg", quantised=False, missing_frac=0.1)
    _check_plan(xgb, wide, Xw, "rows too wide")
    big = P._train(xgb, dict(max_depth=13, min_child_weight=0.5), 16, 3, n=40000, seed=10, slots=True)
    X16, _ = synth(3000, 16, 14, "reg", quantised=False, missing_frac=0.1)
    _check_plan(xgb, big, X16, "tree too large")
    doc = json.loads(bytes(one.bst.save_raw("json")))
    for t in doc["learner"]["gradient_booster"]["model"]["trees"]:
        P._preorder(t)
    _check_plan(xgb, one.reload(json.dumps(doc).encode()), X, "children not adjacent")
    _check_plan(xgb, several, np.ascontiguousarray(X28[:, :20]), "matrix narrower than the model")


# ------------------------------------------------------------------------------------------------------ model kinds
def _kinds(xgb):
    X, y = synth(4000, 12, 21, "reg", quantised=False, missing_frac=0.1)
    Xm, ym = synth(4000, 12, 22, "multi", K=3, quantised=False, missing_frac=0.1)
    yb = (y > 0).astype(np.float32)
    Y2 = np.stack([y, -y * 0.5 + 0.1], axis=1)
    base = dict(tree_method="hist", max_depth=4, eta=0.3)
    out = {
        "binary": (xgb.train(dict(base, objective="binary:logistic"), xgb.DMatrix(X, label=yb), 8), X),
        "softprob": (xgb.train(dict(base, objective="multi:softprob", num_class=3), xgb.DMatrix(Xm, label=ym), 6), Xm),
        "softmax": (xgb.train(dict(base, objective="multi:softmax", num_class=3), xgb.DMatrix(Xm, label=ym), 6), Xm),
        "multi_target": (xgb.train(base, xgb.DMatrix(X, label=Y2), 6), X),
        "quantile": (xgb.train(dict(base, objective="reg:quantileerror", quantile_alpha=[0.2, 0.5, 0.8]), xgb.DMatrix(X, label=y), 6), X),
        "dart": (xgb.train(dict(base, booster="dart", rate_drop=0.3, seed=3), xgb.DMatrix(X, label=y), 8), X),
        "forest": (xgb.train(dict(base, num_parallel_tree=3, subsample=0.7, seed=1), xgb.DMatrix(X, label=y), 5), X),
    }
    qd = xgb.QuantileDMatrix(X, label=y)
    out["quantile_dmatrix"] = (xgb.train(base, qd, 6), X)
    return out


def test_model_kinds(xgb):
    import torch
    for name, (bst, X) in _kinds(xgb).items():
        for ptype in ("value", "margin"):
            kw = dict(output_margin=ptype == "margin")
            for it in ((0, 0), (1, 4)):
                want = _ref(xgb, bst, X, iteration_range=it, **kw)
                _same(bst.inplace_predict(X, predict_type=ptype, iteration_range=it), want)
                _same(bst.inplace_predict(X.astype(np.float64), predict_type=ptype, iteration_range=it), want)
                _same(bst.inplace_predict(torch.from_numpy(X).cuda(), predict_type=ptype, iteration_range=it), want)
            for strict in (False, True):
                want = _ref(xgb, bst, X, strict_shape=strict, **kw)
                _same(bst.inplace_predict(X, predict_type=ptype, strict_shape=strict), want)
        for n in (0, 1):
            _same(bst.inplace_predict(X[:n]), _ref(xgb, bst, X[:n]))
            _same(bst.inplace_predict(torch.from_numpy(X[:n].copy()).cuda()), _ref(xgb, bst, X[:n]))


def test_loaded_model_and_base_margin(xgb):
    import torch
    bst = xgb.Booster(model_file=os.path.join(ROOT, "tests", "golden", "abalone_xgboost-model.ubj"))
    F = bst.num_features()
    X, _ = synth(3000, F, 31, "reg", quantised=False, missing_frac=0.05)
    _same(bst.inplace_predict(X), _ref(xgb, bst, X))
    _same(bst.inplace_predict(X.astype(np.float64), missing=0.0), _ref(xgb, bst, X, missing=0.0))
    Xm, ym = synth(3000, 10, 32, "multi", K=3, quantised=False, missing_frac=0.1)
    multi = xgb.train(dict(tree_method="hist", max_depth=4, objective="multi:softprob", num_class=3), xgb.DMatrix(Xm, label=ym), 5)
    for b, Xb, K in ((bst, X, 1), (multi, Xm, 3)):
        bm = np.random.default_rng(5).standard_normal((Xb.shape[0], K)).astype(np.float32)
        d = xgb.DMatrix(Xb, base_margin=bm.reshape(-1))
        for ptype in ("value", "margin"):
            want = b.predict(d, output_margin=ptype == "margin")
            shaped = bm[:, 0] if K == 1 else bm
            _same(b.inplace_predict(Xb, base_margin=shaped, predict_type=ptype), want)
            _same(b.inplace_predict(torch.from_numpy(Xb).cuda(), base_margin=torch.from_numpy(shaped).cuda(), predict_type=ptype), want)


# ------------------------------------------------------------------------------------------------------ staging
def test_chunked_host_path(xgb, model):
    import torch
    bst, X = model
    be = _be()
    for dtype in ("float32", "float64", "int8", "uint64"):
        A = _cast(X, dtype)
        want = _ref(xgb, bst, A.astype(np.float32))
        try:
            for rows in (7, 1000, 19999):
                be.booster_inplace_debug(bst.handle, rows)
                _same(bst.inplace_predict(A), want)
                _same(bst.inplace_predict(np.asfortranarray(A)), want)
                _same(bst.inplace_predict(torch.from_numpy(A).cuda()), want)
        finally:
            be.booster_inplace_debug(bst.handle, 0)
    for dtype in ("float32", "float64", "float16"):
        bst.inplace_predict(torch.from_numpy(X.astype(dtype)).cuda())
        assert be.booster_inplace_debug(bst.handle)[0] == 0, dtype              # read where it lies: nothing staged
    cap = 32 << 20
    Xl, _ = synth(400000, 28, 41, "reg", quantised=False, missing_frac=0.1)    # 89.6 MB as float64: larger than the cap
    for dtype in ("float64", "int8"):
        A = _cast(Xl, dtype)
        assert A.nbytes > cap or dtype == "int8"
        _same(bst.inplace_predict(A), _ref(xgb, bst, A.astype(np.float32)))
        staged, held = be.booster_inplace_debug(bst.handle)     # a chunk's staged bytes and its float32 conversion, each <= cap
        assert 0 < staged <= (cap if dtype == "float64" else 2 * cap) and held <= 3 * cap, (dtype, staged, held)


# ------------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_booster_usable(xgb, model):
    import torch
    bst, X = model
    want = _ref(xgb, bst, X)
    cases = [lambda: bst.inplace_predict(np.concatenate([X, X], axis=1), validate_features=False),
             lambda: bst.inplace_predict(X.reshape(20000, 14, 2), validate_features=False),
             lambda: bst.inplace_predict(X.astype(np.complex64)),
             lambda: bst.inplace_predict(torch.from_numpy(X).cuda().reshape(20000, 14, 2), validate_features=False)]
    for fn in cases:
        with pytest.raises(xgb.XGBoostError):
            fn()
        _same(bst.inplace_predict(X), want)
    with pytest.raises(ValueError, match="predict_type"):
        bst.inplace_predict(X, predict_type="leaf")
    with pytest.raises(xgb.XGBoostError, match="iteration range"):
        bst.inplace_predict(X, iteration_range=(0, 50))
    _same(bst.inplace_predict(X), want)


def test_cuda_array_on_another_device(xgb, model):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    bst, X = model
    with pytest.raises(xgb.XGBoostError, match="device"):
        bst.inplace_predict(torch.from_numpy(X).to("cuda:1"))
    _same(bst.inplace_predict(X), _ref(xgb, bst, X))


# ------------------------------------------------------------------------------------------------------ C entries
def test_c_entries(xgb, model):
    import torch
    import scipy.sparse as sp
    bst, X = model
    lib = _be().lib
    cfg = json.dumps({"type": 0, "training": False, "iteration_begin": 0, "iteration_end": 0, "strict_shape": False, "missing": float("nan")}).encode()
    shape, dim, res = C.POINTER(C.c_uint64)(), C.c_uint64(), C.POINTER(C.c_float)()
    A = np.asfortranarray(X.astype(np.float64))
    ai = A.__array_interface__
    doc = json.dumps({"data": [ai["data"][0], True], "shape": list(A.shape), "typestr": "<f8", "strides": list(A.strides), "version": 3}).encode()
    assert lib.XGBoosterPredictFromDense(bst.handle, doc, cfg, None, C.byref(shape), C.byref(dim), C.byref(res)) == 0
    got = np.ctypeslib.as_array(res, shape=(shape[0],)).copy()
    _same(got, bst.inplace_predict(A))
    csr = sp.random(500, 28, density=0.4, random_state=2, format="csr", dtype=np.float32)
    ip, ix, dv = csr.indptr.astype(np.int64), csr.indices.astype(np.int32), csr.data
    ifc = lambda a: json.dumps({"data": [a.ctypes.data, True], "shape": list(a.shape), "typestr": a.dtype.str, "version": 3}).encode()
    assert lib.XGBoosterPredictFromCSR(bst.handle, ifc(ip), ifc(ix), ifc(dv), C.c_uint64(28), cfg, None, C.byref(shape), C.byref(dim), C.byref(res)) == 0
    _same(np.ctypeslib.as_array(res, shape=(shape[0],)).copy(), bst.inplace_predict(csr))
    t = torch.from_numpy(X).cuda()
    torch.cuda.synchronize()
    cai = t.__cuda_array_interface__
    doc = json.dumps({"data": [cai["data"][0], False], "shape": list(cai["shape"]), "typestr": "<f4", "strides": None, "version": 3, "stream": None}).encode()
    assert lib.XGBoosterPredictFromCudaArray(bst.handle, doc, cfg, None, C.byref(shape), C.byref(dim), C.byref(res)) == 0
    ptr = C.cast(res, C.c_void_p).value
    out = np.zeros(shape[0], np.float32)
    torch.cuda.synchronize()
    host = torch.empty(shape[0], dtype=torch.float32)
    import sagemaker_xgboost_container_b200.core as core
    host.copy_(torch.as_tensor(core._DeviceResult(ptr, (shape[0],)), device="cuda"))
    out[:] = host.numpy()
    _same(out, _host(bst.inplace_predict(t)))
