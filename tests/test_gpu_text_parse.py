"""The device text parsers (csrc/csv.cu on csrc/text_parse.h) literal for literal and byte for byte, through the backend's own
entry points: dmatrix_from_csv, dmatrix_from_csv_labeled and dmatrix_from_libsvm_text.  Every case asserts the status first
(0 = parsed on the device, 1 = ragged rows, 2 = the host route decides), then the values.

The literal set, the acceptance rule and the reference conversion are those of tests/test_text_parse_sweep.py
(tests/text_parse_reference.py): every literal the rule accepts must come back from the device bit for bit as it comes back
from the host build of parse_field and from encoder.py's numpy conversion -- the device's double arithmetic equals the host's."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import text_parse_reference as R  # noqa: E402
from test_gpu_serving import _ref_dense_route, _ref_sparse_route, _reference_route  # noqa: E402

pytestmark = pytest.mark.gpu


def _csv(xgb, body, delim=","):
    """(status, float32 matrix or None) of the device CSV parse."""
    be = xgb.get_backend()
    h, st = be.dmatrix_from_csv(body, delim)
    if st != 0:
        assert h is None
        return st, None
    d = xgb.DMatrix._from_handle(h)
    return st, be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())


def _libsvm(xgb, body, mode):
    be = xgb.get_backend()
    h, st = be.dmatrix_from_libsvm_text(body, mode, float("nan") if mode == 0 else 0.0)
    if st != 0:
        return st, None
    d = xgb.DMatrix._from_handle(h)
    return st, be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())


@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    work = tmp_path_factory.mktemp("text_parse_gpu")
    lits = R.generate_literals()
    accepted, values = R.run_literals(R.build_helper(work), work, lits)
    return lits, accepted, values


# ------------------------------------------------------------------------------------------------------------ literals
def test_every_fast_path_literal_parses_on_the_device_bit_for_bit(xgb, sweep):
    lits, accepted, host = sweep
    idx = np.nonzero(accepted)[0]
    rule = [R.fast_path_accepts(lits[i]) for i in idx[:20000]]
    assert all(rule)
    want_all = R.reference_float32([lits[i] for i in idx])
    pos, body_no, F = 0, 0, 1
    while pos < len(idx):
        F = body_no % 37 + 1                                              # 1 ... 37 fields per row
        rows, size = [], 0
        while size < 1 << 20 and pos < len(idx):
            take = idx[pos:pos + F]
            if len(take) < F:                                             # fill the last row from the start of the set
                take = np.concatenate([take, idx[:F - len(take)]])
            rows.append(take)
            size += sum(len(lits[i]) + 1 for i in take)
            pos += F
        body = "\n".join(",".join(lits[i] for i in r) for r in rows)
        st, got = _csv(xgb, body)
        assert st == 0, "body %d (F = %d): status %d" % (body_no, F, st)
        order = np.concatenate(rows)
        assert got.shape == (len(rows), F)
        flat = got.reshape(-1)
        assert R.same_float32(flat, host[order]), "body %d differs from the host build of parse_field" % body_no
        pos_in_idx = np.searchsorted(idx, order)
        assert R.same_float32(flat, want_all[pos_in_idx]), "body %d differs from the container's conversion" % body_no
        body_no += 1
    assert body_no > 10


HOST_ROUTE = ["1_000", "0x10", "١٢", "１２", "123456789012345678901234567890", "1e400", "-1e400", "1e-400", "1e23", "9007199254740993",
              "\v1.5", "1.5\f", " ", "\t", "3.4028235e38", "1e39", "0.1000000000000000055511151231257827021181583404541015625"]
MALFORMED = ["e5", "1e", "+", ".", "1.2.3", "--1", "1e5e5", "1e+", "abc", "nan1", "infinit", "1;5", "1 2"]


@pytest.mark.parametrize("lit", HOST_ROUTE + MALFORMED)
def test_literals_outside_the_fast_path_take_the_host_route(xgb, lit):
    from sagemaker_xgboost_container_b200 import serving
    body = "1.5,2,3\n4,%s,6\n7,8,9" % lit
    st, _ = _csv(xgb, body)
    assert st == 2
    try:
        with np.errstate(over="ignore"):
            want = _reference_route(body)
    except Exception as e:                                                # the container's route raises: so must the package
        with pytest.raises(type(e)):
            serving.csv_to_dmatrix(body, dtype=float)
        return
    d = serving.csv_to_dmatrix(body, dtype=float)
    got = xgb.get_backend().dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
    assert R.same_float32(got, want)


def test_generated_literals_outside_the_fast_path_take_the_host_route(xgb, sweep):
    lits, accepted, _ = sweep
    rest = [lits[i] for i in np.nonzero(~accepted)[0] if "," not in lits[i]]
    rng = np.random.default_rng(5)
    for i in rng.choice(len(rest), size=300, replace=False):
        st, _ = _csv(xgb, "1,2\n3,%s\n5,6" % rest[i])
        assert st == 2, repr(rest[i])


# ---------------------------------------------------------------------------------------------------------- body shapes
def _values(rng, n, F):
    return np.where(rng.random((n, F)) < 0.05, np.nan, rng.standard_normal((n, F)) * 10.0 ** rng.integers(-5, 6, size=(n, F)))


def _body(X, delim=","):
    return "\n".join(delim.join("" if v != v else "%.7g" % v for v in row) for row in X)


def _check(xgb, body, delim=","):
    st, got = _csv(xgb, body, delim)
    assert st == 0
    assert R.same_float32(got, _reference_route(body, delim))


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65537])
def test_row_counts(xgb, n):
    _check(xgb, _body(_values(np.random.default_rng(n), n, 3)))


def test_one_row_of_5000_fields(xgb):
    _check(xgb, _body(_values(np.random.default_rng(1), 1, 5000)))


@pytest.mark.parametrize("rem", [0, 1, 15])
def test_body_length_around_the_16_byte_vectors(xgb, rem):
    for n in (1, 2, 40):
        body = _body(_values(np.random.default_rng(n), n, 4))
        pad = (rem - len(body)) % 16
        body = "0" * pad + body                                          # leading zeros of the first field
        assert len(body) % 16 == rem
        _check(xgb, body)


def test_trailing_newline_delimiter_and_empty_fields(xgb):
    _check(xgb, "1\n2\n")                                               # F = 1: the last row is one empty field (NaN)
    assert _csv(xgb, "1,2\n3,4\n")[0] == 1                               # F > 1: the empty last row is ragged
    with pytest.raises(ValueError):
        _reference_route("1,2\n3,4\n")
    _check(xgb, "1,2,\n3,4,")                                          # trailing delimiter: an empty last field
    _check(xgb, ",1\n,2")
    _check(xgb, "1,\n2,")
    _check(xgb, ",\n,")


@pytest.mark.parametrize("delim", [",", ";", "\t", "|", " "])
def test_delimiters(xgb, delim):
    X = _values(np.random.default_rng(ord(delim)), 300, 7)
    _check(xgb, _body(X, delim), delim)


@pytest.mark.parametrize("body", ["1,2,3\n4,5", "1,2\n3,4,5", "1\n2,3", "1,2\n\n3,4", "1,2\n3,4\n5"])
def test_ragged_bodies(xgb, body):
    assert _csv(xgb, body)[0] == 1
    with pytest.raises(ValueError):
        _reference_route(body)


# ---------------------------------------------------------------------------------------------------- newline byte sweep
def _predicted_status(body, F):
    """csv_parse_kernel's status from the fast-path rule: 2 if a field it parses is not taken, else 1 if a row is ragged."""
    st = 0
    for row in body.split(b"\n"):
        fields = row.split(b",")
        if len(fields) != F:
            st = max(st, 1)
        if not all(R.fast_path_accepts(f.decode("latin-1")) for f in fields[:F]):
            st = 2
    return st


def test_every_byte_after_a_newline_at_every_offset(xgb):
    tail = b"\n3.25,-4\n5,6e-3\n7,8"
    for off in range(16):
        first = b"0" * off + b"1,2"                                       # the first '\n' lands at offset off + 3 (mod 16)
        for b in range(256):
            body = first + b"\n" + bytes([b]) + b"9,10" + tail
            st, got = _csv(xgb, body)
            assert st == _predicted_status(body, 2), (off, b)
            if st == 0:
                want = _reference_route(body.decode("ascii"))
                assert got.shape == want.shape and R.same_float32(got, want), (off, b)


@pytest.mark.parametrize("ws", ["\v", "\f", "\t", "\r", " "])
def test_libsvm_whitespace_after_a_newline(xgb, ws):
    for off in range(16):
        body = "1" + " " * off + " 1:2\n" + ws + "0 2:3\n1 3:0.5"
        st, got = _libsvm(xgb, body, 1)
        assert st == 0, (off, ws)
        want = _ref_dense_route(body)
        assert got.shape == want.shape and R.same_float32(got, want), (off, ws)


def test_scratch_is_not_reused_across_bodies(xgb):
    big = _body(_values(np.random.default_rng(9), 200_000, 5))
    _check(xgb, big)
    body = "1 1:2\n\v0 2:3"
    st, got = _libsvm(xgb, body, 1)
    assert st == 0 and got.shape == (2, 2) and R.same_float32(got, _ref_dense_route(body))
    st, got = _libsvm(xgb, body, 0)
    assert st == 0 and R.same_float32(got, _ref_sparse_route(body))
    _check(xgb, "1,2\n3,4")
    _check(xgb, "5")


# ----------------------------------------------------------------------------------------------------- training channels
@pytest.mark.parametrize("label,weight", [(0, -1), (0, 1), ("last", 0), (2, 1)])
def test_training_channel_label_and_weight_columns(xgb, label, weight):
    rng = np.random.default_rng(11)
    n, F = 5000, 6
    label = F - 1 if label == "last" else label
    X = (rng.standard_normal((n, F)) * 10.0 ** rng.integers(-6, 7, size=(n, F))).astype(np.float32)
    if weight >= 0:
        X[:, weight] = np.abs(X[:, weight])                              # weights must not be negative
    fields = [["%.9g" % v for v in row] for row in X]
    for r in range(0, n, 37):
        if (r // 37) % F != weight:
            fields[r][(r // 37) % F] = ["-0", "1e-22", "inf", "12345678", ".5", "7."][r % 6]
    body = "\n".join(",".join(row) for row in fields).encode("ascii")
    be = xgb.get_backend()
    h, st = be.dmatrix_from_csv_labeled(body, ",", label, weight)
    assert st == 0
    d = xgb.DMatrix._from_handle(h)
    ref = np.array([[float(v) for v in row] for row in fields], dtype=np.float64).astype(np.float32)
    keep = [c for c in range(F) if c not in (label, weight)]
    got = be.dmatrix_get_raw(d.handle).reshape(d.num_row(), d.num_col())
    assert R.same_float32(got, ref[:, keep])
    assert R.same_float32(d.get_label(), ref[:, label])
    if weight >= 0:
        assert R.same_float32(d.get_weight(), ref[:, weight])


def test_training_channel_label_equal_to_weight_raises(xgb):
    with pytest.raises(xgb.XGBoostError):
        xgb.get_backend().dmatrix_from_csv_labeled(b"1,2,3\n4,5,6", ",", 1, 1)
