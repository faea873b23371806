"""recordio-protobuf bodies decoded on the device (csrc/recordio.cu) against the container's own reader: the goldens of
tests/golden/make_recordio_goldens.py (the reference's 12 fixtures and seeded random bodies), large seeded bodies against the
numpy matrix they encode, training from a channel directory and serving a request.  Needs neither the reference nor protobuf."""
import os

import numpy as np
import pytest

import recordio_reference as R
import sagemaker_xgboost_container_b200 as xgb
from sagemaker_xgboost_container_b200 import data, recordio, serving
from sagemaker_xgboost_container_b200.backend import get_backend

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(R.GOLDEN_DIR, "decoded.npz"))


def _raw(d):
    return get_backend().dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())


def _check(key, body, statuses):
    """The device decode of `body` equals golden `key`: the matrix and label bit for bit, or the same error."""
    be = get_backend()
    h, status, message = be.dmatrix_from_recordio(body)
    statuses[status] += 1
    if key + "_error" in GOLDEN.files:
        assert str(GOLDEN[key + "_error"]) == "ValueError"
        if status == 1:
            assert message
        with pytest.raises(ValueError):
            recordio.recordio_protobuf_to_dmatrix(body)
        assert status != 0, key
        return
    assert status != 1, (key, message)
    d = xgb.DMatrix._from_handle(h) if status == 0 else recordio.recordio_protobuf_to_dmatrix(body)
    want = GOLDEN[key + "_X"]
    got = _raw(d)
    assert got.shape == want.shape, key
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), key
    assert np.array_equal(d.get_label().view(np.uint32), GOLDEN[key + "_label"].view(np.uint32)), key


def test_fixtures_match_goldens():
    statuses = {0: 0, 1: 0, 2: 0}
    for i, name in enumerate(R.FIXTURES):
        assert str(GOLDEN["fixture%d_name" % i]) == name
        with open(os.path.join(R.GOLDEN_DIR, name.replace("/", "__")), "rb") as f:
            _check("fixture%d" % i, f.read(), statuses)
    assert statuses == {0: 9, 1: 3, 2: 0}, statuses


def test_random_bodies_match_goldens():
    statuses = {0: 0, 1: 0, 2: 0}
    for seed in range(R.N_RANDOM):
        body = R.random_body(seed)
        assert R.body_digest(body) == str(GOLDEN["random%d_body_sha256" % seed]), seed
        _check("random%d" % seed, body, statuses)
    assert statuses[0] >= R.N_RANDOM // 2 and statuses[1] >= 10 and statuses[2] >= 10, statuses


@pytest.mark.parametrize("n,F,kind", [(2_000_000, 28, "f32"), (300_000, 28, "f64"), (20_000, 1500, "f32"), (3, 1100, "f64")])
def test_large_dense_bodies(n, F, kind):
    body, X, y = R.big_dense_body(n, F, seed=n + F, kind=kind)
    d = serving.recordio_protobuf_to_dmatrix(body)
    assert np.array_equal(_raw(d).view(np.uint32), X.view(np.uint32))
    assert np.array_equal(d.get_label(), y)


@pytest.mark.parametrize("n,F,k", [(2_000_000, 100, 10), (100_000, 127, 127), (1000, 5, 1)])
def test_large_sparse_bodies(n, F, k):
    body, X, y = R.big_sparse_body(n, F, k, seed=n + k)
    d = serving.recordio_protobuf_to_dmatrix(bytearray(body))
    assert np.array_equal(_raw(d).view(np.uint32), X.view(np.uint32))
    assert np.array_equal(d.get_label(), y)


def test_train_from_channel_and_serve(tmp_path):
    body, X, y = R.big_dense_body(30_000, 12, seed=3)
    rec_len = len(body) // 30_000
    cuts = [0, 7_000, 19_000, 30_000]
    for i in range(3):                                     # three data files, plus files the channel reader skips
        (tmp_path / ("part-%d.pbr" % i)).write_bytes(body[cuts[i] * rec_len:cuts[i + 1] * rec_len])
    (tmp_path / ".hidden").write_bytes(b"junk")
    (tmp_path / "_SUCCESS").write_bytes(b"")
    (tmp_path / "dtrain.cache.page").write_bytes(b"junk")
    d = data.recordio_protobuf_to_dmatrix(str(tmp_path))
    params = dict(objective="binary:logistic", tree_method="hist", max_depth=5, eta=0.3, max_bin=64)
    a = xgb.train(params, d, num_boost_round=4)
    b = xgb.train(params, xgb.DMatrix(X, label=y), num_boost_round=4)
    assert bytes(a.save_raw("ubj")) == bytes(b.save_raw("ubj"))
    request = body[:500 * rec_len]
    got = serving.predict(a, "ubj", serving.recordio_protobuf_to_dmatrix(request), "application/x-recordio-protobuf")
    assert np.array_equal(got, b.predict(xgb.DMatrix(X[:500])))
    empty = tmp_path / "empty"
    empty.mkdir()
    assert data.recordio_protobuf_to_dmatrix(str(empty)) is None
    with pytest.raises(xgb.XGBoostError):
        data.recordio_protobuf_to_dmatrix(str(tmp_path), is_pipe=True)


def test_host_route_bodies_decode_identically():
    """Bodies with encodings the device path hands back (status 2) give what their plain encoding gives on the device."""
    be = get_backend()
    rng = np.random.default_rng(11)
    vals = rng.standard_normal((40, 6)).astype(np.float32)
    plain = R.frame([R.record([("values", R.value("f32", R.tensor("f32", v)))], [("values", R.value("i32", R.tensor("i32", [i])))])
                     for i, v in enumerate(vals)])
    variants = {
        "unpacked": [R.record([("values", R.value("f32", R.tensor("f32", v, packed=False)))], [("values", R.value("i32", R.tensor("i32", [i])))])
                     for i, v in enumerate(vals)],
        "merged": [R.record([("values", R.value("f32", R.tensor("f32", v[:2])) + R.value("f32", R.tensor("f32", v[2:])))],
                            [("values", R.value("i32", R.tensor("i32", [i])))]) for i, v in enumerate(vals)],
        "repeated_key": [R.record([("values", R.value("f32", R.tensor("f32", [7.0]))), ("values", R.value("f32", R.tensor("f32", v)))],
                                  [("values", R.value("i32", R.tensor("i32", [i])))]) for i, v in enumerate(vals)],
    }
    h, status, _ = be.dmatrix_from_recordio(plain)
    assert status == 0
    want = xgb.DMatrix._from_handle(h)
    for name, recs in variants.items():
        body = R.frame(recs)
        assert be.dmatrix_from_recordio(body)[1] == 2, name
        got = recordio.recordio_protobuf_to_dmatrix(body)
        assert np.array_equal(_raw(got).view(np.uint32), _raw(want).view(np.uint32)), name
        assert np.array_equal(got.get_label(), want.get_label()), name


def test_reference_errors_raise():
    ok = R.record([("values", R.value("f32", R.tensor("f32", [1.0, 2.0])))])
    for body, words in ((R.frame([ok])[:-3], "Truncated"), (b"\x00" * 8 + R.frame([ok]), "magic"), (b"", "No records"),
                        (R.frame([ok, R.record([("values", R.value("f32", R.tensor("f32", [1.0])))])]), "lengths")):
        with pytest.raises(ValueError, match=words):
            serving.recordio_protobuf_to_dmatrix(body)
    assert serving.recordio_protobuf_to_dmatrix(R.frame([ok], trailing=b"\1" * 7)).num_row() == 1
