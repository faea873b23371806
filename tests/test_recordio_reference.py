"""The package's host decoder of recordio-protobuf bodies (sagemaker_xgboost_container_b200.recordio.read_recordio_protobuf, the
route the device path hands odd encodings to) against the container's own `read_recordio_protobuf`, run unchanged with
`sagemaker_containers.record_pb2` stubbed by a Record class built from descriptors.  Skips where the reference checkout or
google.protobuf is absent.  Needs no GPU."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import recordio_reference as R
from sagemaker_xgboost_container_b200 import recordio

pytestmark = pytest.mark.skipif(not R.reference_available(), reason="needs the reference checkout and google.protobuf")


@pytest.fixture(scope="module")
def reference():
    return R.reference_reader()


def _outcome(fn, body):
    try:
        return fn(body)
    except Exception as e:
        return type(e)


def _same(a, b):
    if isinstance(a, type) or isinstance(b, type):
        assert a is b or (isinstance(a, type) and isinstance(b, type) and issubclass(a, ValueError) and issubclass(b, ValueError)), (a, b)
        return
    (fa, la), (fb, lb) = a, b
    assert sp.issparse(fa) == sp.issparse(fb)
    assert fa.shape == fb.shape and fa.dtype == fb.dtype
    if sp.issparse(fa):
        for attr in ("indptr", "indices"):
            assert np.array_equal(getattr(fa, attr), getattr(fb, attr))
        assert np.array_equal(fa.data.view(np.uint8), fb.data.view(np.uint8))
    else:
        assert np.array_equal(np.ascontiguousarray(fa).view(np.uint8), np.ascontiguousarray(fb).view(np.uint8))
    assert (la is None) == (lb is None)
    if la is not None:
        assert la.dtype == lb.dtype and np.array_equal(la.view(np.uint8), lb.view(np.uint8))


@pytest.mark.parametrize("name", R.FIXTURES)
def test_fixture_matches_reference(reference, name):
    with open(os.path.join(R.REFERENCE_FIXTURES, name), "rb") as f:
        body = f.read()
    read, _ = reference
    _same(_outcome(recordio.read_recordio_protobuf, body), _outcome(read, body))


def test_random_bodies_match_reference(reference):
    read, _ = reference
    kinds = {"ok_dense": 0, "ok_sparse": 0, "error": 0}
    for seed in range(R.N_RANDOM):
        body = R.random_body(seed)
        ours, ref = _outcome(recordio.read_recordio_protobuf, body), _outcome(read, body)
        _same(ours, ref)
        kinds["error" if isinstance(ref, type) else ("ok_sparse" if sp.issparse(ref[0]) else "ok_dense")] += 1
    assert min(kinds.values()) >= 20, kinds        # every outcome is exercised


def test_reference_fixture_table(reference):
    """What the reference gives on its fixtures, as DESIGN.md records it."""
    read, _ = reference

    def load(name):
        with open(os.path.join(R.REFERENCE_FIXTURES, name), "rb") as f:
            return f.read()
    X, y = read(load("train.pb"))
    assert isinstance(X, np.ndarray) and X.shape == (5, 5) and X.dtype == np.int32 and y.dtype == np.int32
    X, y = read(load("single_feature_label.pb"))
    assert X.shape == (1, 0) and len(y) == 1
    assert read(load("sparse/train.pb"))[0].shape == (5, 5)
    assert read(load("sparse_edge_cases/rectangular_sparse.pbr"))[0].shape == (4, 3)
    for k in ("center", "top_left", "top_right"):
        with pytest.raises(ValueError):
            read(load("sparse_edge_cases/single_value_%s.pbr" % k))


def test_encoder_matches_protobuf(reference):
    """The test's own encoder writes what google.protobuf serialises (deterministic map order = keys sorted)."""
    _, Record = reference
    rng = np.random.default_rng(7)
    for i in range(60):
        kind = ["f32", "f64", "i32"][i % 3]
        vals = R._vals(rng, kind, int(rng.integers(0, 6)))
        keys = rng.integers(0, 1 << int(rng.integers(1, 63)), int(rng.integers(0, 4)), dtype=np.uint64) if i % 2 else []
        shape = [int(rng.integers(0, 300))] if i % 4 < 2 else []
        r = Record()
        t = getattr(r.features["values"], {"f32": "float32_tensor", "f64": "float64_tensor", "i32": "int32_tensor"}[kind])
        t.values.extend(vals.tolist())
        t.keys.extend(int(k) for k in keys)
        t.shape.extend(shape)
        r.label["values"].float64_tensor.values.append(float(i))
        if i % 5 == 0:
            r.features["zz"].bytes.value.append(b"abc")
        if i % 7 == 0:
            r.uid = "u%d" % i
        feats = [("values", R.value(kind, R.tensor(kind, vals, keys, shape)))]
        if i % 5 == 0:
            feats.append(("zz", R.value(raw=b"abc")))
        ours = R.record(feats, [("values", R.value("f64", R.tensor("f64", [float(i)])))], uid="u%d" % i if i % 7 == 0 else None)
        assert ours == r.SerializeToString(deterministic=True), i


def test_host_route_handles_what_the_device_hands_back(reference):
    """Encodings the device path leaves to the host route decode as protobuf decodes them."""
    read, Record = reference
    vals = [1.5, 0.0, -2.0]
    odd = [
        R.record([("values", R.value("f32", R.tensor("f32", vals, packed=False)))]),                      # unpacked values
        R.record([("values", R.value("f32", R.tensor("f32", vals[:1])) + R.value("f32", R.tensor("f32", vals[1:])))]),  # merged tensors
        R.record([("values", R.value("f32", R.tensor("f32", [9.0]))), ("values", R.value("f32", R.tensor("f32", vals)))]),  # repeated key
        R.record([("values", R.value("i32", R.tensor("i32", [1, 2])) + R.value("f64", R.tensor("f64", [3.0, 4.0, 5.0])))]),  # oneof switch
    ]
    for payload in odd:
        body = R.frame([payload, payload])
        _same(_outcome(recordio.read_recordio_protobuf, body), _outcome(read, body))
