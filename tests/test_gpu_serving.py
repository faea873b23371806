"""Serving input path on the device (BASELINE config 5; SURVEY.md section 8f row 1): the CSV request body parsed by csv.cu must
give exactly the float32 matrix the container's own route builds (encoder.csv_to_dmatrix: str.split -> np.array -> float64 ->
DMatrix float32), for every literal form Python's float() accepts; anything outside the exact fast path falls back to it."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _reference_route(payload, delimiter=","):
    rows = [["nan" if x == "" else x for x in line.split(delimiter)] for line in payload.split("\n")]      # encoder.py:31-32,50
    return np.array(rows).astype(float).astype(np.float32)                                                # xgb.DMatrix(float64) stores float32


def _device_matrix(xgb, payload):
    from sagemaker_xgboost_container_b200 import serving
    d = serving.csv_to_dmatrix(payload, dtype=float)
    n, F = d.num_row(), d.num_col()
    be = xgb.get_backend()
    return be.dmatrix_get_raw(d.handle).reshape(n, F), d


def _mixed_body(formats, specials, seed=7):
    rng = np.random.default_rng(seed)
    n, F = 20000, 28
    X = rng.standard_normal((n, F)) * np.exp(rng.uniform(-20, 20, size=(n, F)))
    lines = []
    for r in range(n):
        fmt = formats[r % len(formats)]
        vals = [(fmt % (int(v) if fmt == "%d" else v)) for v in X[r]]
        if r % 97 == 0:
            vals[r % F] = ""                     # empty field -> NaN
        if r % 101 == 0:
            vals[(r + 3) % F] = specials[(r // 101) % len(specials)]
        lines.append(",".join(vals))
    return "\n".join(lines)


def _assert_same(got, ref):
    assert got.shape == ref.shape
    assert np.array_equal(got.view(np.uint32)[~np.isnan(ref)], ref.view(np.uint32)[~np.isnan(ref)])          # bit-exact, incl. -0, inf
    assert np.array_equal(np.isnan(got), np.isnan(ref))


def test_csv_payload_device_parse_is_bit_identical_to_the_container_route(xgb):
    """Every field inside the exact fast path: the device must take the whole body (status 0), not hand it to the host route."""
    payload = _mixed_body(["%.6g", "%.9g", "%.3e", "%d", "%.4f"], ["nan", "NaN", "inf", "-inf", "+1.5", " 2.5 ", "-0", "1e-22", "1E+05", ".5"])
    be = xgb.get_backend()
    h, st = be.dmatrix_from_csv(payload, ",")
    assert st == 0
    d = xgb.DMatrix._from_handle(h)
    _assert_same(be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col()), _reference_route(payload))


def test_csv_payload_outside_the_fast_path_takes_the_host_route_bit_identically(xgb):
    """%.17g and %.9f fields (mantissas >= 2^53, exponents beyond +-22) and literals that overflow float32: status 2 on the
    device, then the container's own route through serving.csv_to_dmatrix."""
    payload = _mixed_body(["%.6g", "%.17g", "%.3e", "%d", "%.9f"], ["nan", "inf", "-0", "1e-45", "3.4028235e38", "1e39"])
    h, st = xgb.get_backend().dmatrix_from_csv(payload, ",")
    assert st == 2 and h is None
    got, _ = _device_matrix(xgb, payload)
    with np.errstate(over="ignore"):
        _assert_same(got, _reference_route(payload))


def test_csv_semicolon_single_row_and_single_column(xgb):
    for payload in ("1.5;2;;4", "3.25", "1\n2\n3", "1e3,2e-3\n-4,5"):
        delim = ";" if ";" in payload else ","
        got, _ = _device_matrix(xgb, payload)
        ref = _reference_route(payload, delim)
        np.testing.assert_array_equal(np.nan_to_num(got, nan=-777.0), np.nan_to_num(ref, nan=-777.0))


def test_csv_out_of_fast_path_literals_fall_back_to_the_host_route(xgb):
    payload = "0.1000000000000000055511151231257827021181583404541015625,2\n123456789012345678901234567890,1e400"
    got, _ = _device_matrix(xgb, payload)
    ref = _reference_route(payload)
    np.testing.assert_array_equal(got, ref)


def test_csv_ragged_and_malformed_payloads_raise(xgb):
    from sagemaker_xgboost_container_b200 import serving
    with pytest.raises(ValueError):
        serving.csv_to_dmatrix("1,2,3\n4,5", dtype=float)
    with pytest.raises(ValueError):
        serving.csv_to_dmatrix("1,2\n3,abc", dtype=float)


def test_serving_predict_matches_direct_predict(xgb):
    from sagemaker_xgboost_container_b200 import serving
    from util import synth
    X, y = synth(5000, 12, 3, "bin")
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(dict(objective="binary:logistic", max_depth=4), d, num_boost_round=5, verbose_eval=False)
    payload = "\n".join(",".join("%.9g" % v for v in row) for row in X[:300])
    dtest = serving.csv_to_dmatrix(payload, dtype=float)
    p = serving.predict(bst, "xgb_format", dtest, "text/csv", objective="binary:logistic")
    np.testing.assert_array_equal(p, bst.predict(xgb.DMatrix(X[:300])))
    ens = serving.predict([bst, bst], ["xgb_format"] * 2, dtest, "text/csv", objective="binary:logistic")
    np.testing.assert_allclose(ens, p, rtol=0, atol=1e-7)


def test_training_csv_channel_is_parsed_on_the_device_like_the_host_loader(xgb, tmp_path):
    """data_utils.py:289-318: a directory of CSV files, label in column 0, optional weight in column 1 (csv_weights=1)."""
    from sagemaker_xgboost_container_b200.data import load_uri
    rng = np.random.default_rng(3)
    d = tmp_path / "train"
    d.mkdir()
    for i in range(3):
        A = np.round(rng.standard_normal((700 + i, 9)) * 10.0 ** rng.integers(-3, 4, size=(1, 9)), 5)
        A[:, 1] = np.abs(A[:, 1]) + 0.5          # weights must be non-negative
        lines = [",".join("" if (r + c) % 53 == 0 and c > 1 else repr(float(v)) for c, v in enumerate(row)) for r, row in enumerate(A)]
        (d / ("part-%d.csv" % i)).write_text("\n".join(lines) + "\n")
    uri = "%s?format=csv&label_column=0&delimiter=,&weight_column=1" % d
    dm = xgb.DMatrix(uri)
    X, y, w = load_uri(uri)                      # host loader (pandas' C parser: its fast strtod may be 1 ulp off in double)
    be = xgb.get_backend()
    got = be.dmatrix_get_raw(dm.handle).reshape(dm.num_row(), dm.num_col())
    assert got.shape == X.shape
    # exact reference: Python's correctly rounded float() of every field, then float32 -- the device parser must match it bit for bit
    rows = [l.split(",") for f in sorted(os.listdir(d)) for l in open(d / f).read().strip().split("\n")]
    ref = np.array([[np.nan if v == "" else float(v) for v in r] for r in rows], dtype=np.float64).astype(np.float32)
    np.testing.assert_array_equal(np.nan_to_num(got, nan=-777.0), np.nan_to_num(ref[:, 2:], nan=-777.0))
    np.testing.assert_array_equal(dm.get_label(), ref[:, 0])
    np.testing.assert_array_equal(dm.get_weight(), ref[:, 1])
    np.testing.assert_allclose(np.nan_to_num(got, nan=-777.0), np.nan_to_num(X, nan=-777.0), rtol=2e-7, atol=0)
    np.testing.assert_allclose(dm.get_label(), y, rtol=2e-7)


# ------------------------------------------------------------------------------------------------ libsvm request bodies
def _ref_sparse_route(payload):
    """serve_utils._get_sparse_matrix_from_libsvm + xgb.DMatrix(csr) (algorithm_mode/serve_utils.py:94-118,132-137), restated"""
    from scipy.sparse import csr_matrix
    row, col, data = [], [], []
    for r, line in enumerate(x.split(" ") for x in payload.split("\n")):
        for item in line:
            if ":" in item:
                col.append(int(item.split(":")[0])); row.append(r); data.append(item.split(":")[1])
    row, col = np.array(row), np.array(col).astype(int)
    if len(col) > 0 and col.min() >= 1:
        col = col - 1
    m = csr_matrix((np.array(data).astype(float), (row, col)))
    out = np.full(m.shape, np.nan, np.float32)
    coo = m.tocoo()
    out[coo.row, coo.col] = coo.data.astype(np.float32)
    return out


def _ref_dense_route(payload):
    """encoder.libsvm_to_dmatrix (encoder.py:54-86), restated"""
    rows = []
    for line in payload.strip().split("\n"):
        row = {}
        for token in line.strip().split():
            if ":" in token:
                idx, val = token.split(":", 1)
                row[int(idx)] = float(val)
        rows.append(row)
    mn = min(i for r in rows for i in r)
    off = 1 if mn >= 1 else 0
    data = np.zeros((len(rows), max(i for r in rows for i in r) - off + 1))
    for i, r in enumerate(rows):
        for k, v in r.items():
            data[i, k - off] = v
    return data.astype(np.float32)


def _libsvm_body(rng, n, F, one_based=True, fmt="%.6g"):
    lines = []
    for r in range(n):
        k = int(rng.integers(0, F + 1)) if r not in (0, n - 1) else max(1, int(rng.integers(1, F + 1)))
        idx = np.sort(rng.choice(F, size=k, replace=False))
        if r == 0:
            idx = np.union1d(idx, [0])                                    # the smallest index decides the 1-based shift: pin it
        idx = idx + (1 if one_based else 0)
        vals = rng.standard_normal(len(idx)) * np.exp(rng.uniform(-10, 10, len(idx)))
        toks = ["%d" % int(rng.integers(0, 3))] + ["%d:%s" % (i, (fmt % v) if j % 7 else "%d" % int(v)) for j, (i, v) in enumerate(zip(idx, vals))]
        lines.append(" ".join(toks))
    return "\n".join(lines)


@pytest.mark.parametrize("one_based", [True, False])
def test_libsvm_bodies_on_the_device_match_both_container_routes(xgb, one_based):
    from sagemaker_xgboost_container_b200 import serving
    rng = np.random.default_rng(31 + one_based)
    body = _libsvm_body(rng, 5000, 40, one_based)
    be = xgb.get_backend()
    h, st = be.dmatrix_from_libsvm_text(body, 0, float("nan"))
    assert st == 0                                                        # the fast path took it (no silent host fallback in this test)
    d = xgb.DMatrix._from_handle(h)
    want = _ref_sparse_route(body)
    got = be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
    assert got.shape == want.shape and got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()
    h, st = be.dmatrix_from_libsvm_text(body, 1, 0.0)
    assert st == 0
    d = xgb.DMatrix._from_handle(h)
    want = _ref_dense_route(body)
    got = be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
    assert got.shape == want.shape and got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()
    d2 = serving.sparse_libsvm_to_dmatrix(body)
    assert (d2.num_row(), d2.num_col()) == _ref_sparse_route(body).shape


@pytest.mark.parametrize("body,why", [
    ("1 1:0.5 1:0.25 2:3", "index repeated inside a line (COO sums, dict keeps the last)"),
    ("1 1:0.5 2:3\n0\n", "trailing line without entries"),
    ("1 +1:0.5 2:3", "index that is not plain digits"),
    ("1 1:0.12345678901234567890123 2:3", "literal outside the exact fast path"),
    ("1 1:nan 2:3", "NaN value"),
    ("1 1:2\t3:4 5:6", "tab inside a token"),
])
def test_libsvm_special_cases_take_the_host_route_and_agree(xgb, body, why):
    from sagemaker_xgboost_container_b200 import serving
    be = xgb.get_backend()
    h, st = be.dmatrix_from_libsvm_text(body.strip(), 0, float("nan"))
    assert st == 2 and h is None, why
    try:
        want = _ref_sparse_route(body.strip())
    except Exception as e:                                               # the reference raises: so must the mirror
        with pytest.raises(type(e)):
            serving.sparse_libsvm_to_dmatrix(body.strip())
        return
    d = serving.sparse_libsvm_to_dmatrix(body.strip())
    got = be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
    np.testing.assert_array_equal(got, want)


def test_libsvm_dense_route_edge_cases(xgb):
    from sagemaker_xgboost_container_b200 import serving
    be = xgb.get_backend()
    for body in ["1 1:0.5 1:0.25 2:3\n0\n1 4:1", "0 3:1e-3\t7:2 \n\n1 1:5", "1 0:1 5:2\n0 2:3"]:
        d = serving.libsvm_to_dmatrix(body)
        want = _ref_dense_route(body)
        got = be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
        assert got.shape == want.shape and got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes(), body
    assert serving.libsvm_to_dmatrix("1\n0\n").num_row() == 0            # no entry at all: the reference's empty DMatrix
