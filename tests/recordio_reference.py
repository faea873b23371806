"""recordio-protobuf test support, shared by tests/test_recordio_reference.py, tests/test_gpu_recordio.py and
tests/golden/make_recordio_goldens.py:

  * a wire-format encoder of the aialgs.data Record schema in plain Python (no google.protobuf needed),
  * seeded random bodies that cover the decoding rules (DESIGN.md "recordio-protobuf"), and large seeded bodies with the numpy
    matrix they hold,
  * where google.protobuf and the reference checkout exist: the reference's own `read_recordio_protobuf`, imported with
    `sagemaker_containers.record_pb2` stubbed by a Record class built from descriptors.
"""
import hashlib
import importlib.util
import os
import struct
import sys
import types

import numpy as np

from reference_stubs import REFERENCE_SRC

MAGIC = 0xCED7230A
TENSOR_FIELD = {"f32": 2, "f64": 3, "i32": 7}
REFERENCE_FIXTURES = os.path.join(os.path.dirname(REFERENCE_SRC), "test", "resources", "data", "recordio_protobuf")
FIXTURES = ["train.pb", "pb_files/train.pb", "sparse/train.pb", "single_feature_label.pb"] + [
    "sparse_edge_cases/%s.pbr" % k for k in ("dense_as_sparse", "diagonal", "rectangular_sparse", "single_value_bot_left", "single_value_bot_right",
                                             "single_value_center", "single_value_top_left", "single_value_top_right")]
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recordio")
N_RANDOM = 240


# ------------------------------------------------------------------------------------------------------------- encoder
def varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def tag(field, wire_type):
    return varint(field << 3 | wire_type)


def ld(field, payload):
    return tag(field, 2) + varint(len(payload)) + payload


def _scalars(kind, values):
    if kind == "f32":
        return [struct.pack("<I", int(u)) for u in np.asarray(values, np.float32).view(np.uint32)]
    if kind == "f64":
        return [struct.pack("<Q", int(u)) for u in np.asarray(values, np.float64).view(np.uint64)]
    return [varint(int(v)) for v in np.asarray(values, np.int64)]          # int32: negative values take 10 bytes


def tensor(kind, values=(), keys=(), shape=(), packed=True):
    """A Float32Tensor / Float64Tensor / Int32Tensor message; packed=False writes every value / key with its own tag."""
    out = b""
    if len(values):
        items = _scalars(kind, values)
        if packed:
            out += ld(1, b"".join(items))
        else:
            wt = {"f32": 5, "f64": 1, "i32": 0}[kind]
            out += b"".join(tag(1, wt) + it for it in items)
    for field, arr in ((2, keys), (3, shape)):
        if len(arr):
            if packed:
                out += ld(field, b"".join(varint(int(k)) for k in arr))
            else:
                out += b"".join(tag(field, 0) + varint(int(k)) for k in arr)
    return out


def value(kind=None, tensor_bytes=b"", raw=None):
    """A Value: the tensor of `kind`, raw bytes (field 9, a Bytes message) when raw is given, nothing set when both are None."""
    if raw is not None:
        return ld(9, ld(1, raw))
    if kind is None:
        return b""
    return ld(TENSOR_FIELD[kind], tensor_bytes)


def map_entry(key, value_bytes):
    return ld(1, key.encode() if isinstance(key, str) else key) + ld(2, value_bytes)


def record(features=(), label=(), uid=None, extra=b""):
    """A Record: features / label are lists of (key, Value bytes), in the order they are written."""
    out = b"".join(ld(1, map_entry(k, v)) for k, v in features)
    out += b"".join(ld(2, map_entry(k, v)) for k, v in label)
    if uid is not None:
        out += ld(3, uid.encode())
    return out + extra


def frame(payloads, trailing=b""):
    out = bytearray()
    for p in payloads:
        out += struct.pack("<II", MAGIC, len(p)) + p + b"\0" * (-len(p) % 4)
    return bytes(out + trailing)


def body_digest(body):
    return hashlib.sha256(body).hexdigest()


# ------------------------------------------------------------------------------------------------------------- random bodies
_SPECIAL = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-40, -3e-39, 1.5, -2.25, 16777217.0, 3.4e38, 1e-310], np.float64)


def _vals(rng, kind, n):
    if kind == "i32":
        pool = np.array([0, 1, -1, 7, -7, 16777217, -16777219, 2**31 - 1, -2**31, 123456789], np.int64)
        v = rng.integers(-1000, 1000, n)
        pick = rng.random(n) < 0.3
        v[pick] = rng.choice(pool, pick.sum())
        return v
    v = np.round(rng.standard_normal(n) * 8, 2)
    pick = rng.random(n) < 0.3
    v[pick] = rng.choice(_SPECIAL, pick.sum())
    if kind == "f64":
        v[rng.random(n) < 0.1] = 0.1 + 1e-12
    return v


def random_body(seed):
    """A seeded body for the host-route / device comparisons: mode = seed % 4 picks dense, sparse, mixed or odd encodings."""
    rng = np.random.default_rng(1000 + seed)
    mode = seed % 4
    n = int(rng.integers(1, 10))
    width = int(rng.integers(0, 7)) if mode == 0 else int(rng.integers(1, 9))
    body_kind = ["f32", "f64", "i32"][int(rng.integers(0, 3))]
    odd = mode == 3
    recs = []
    for _ in range(n):
        kind = body_kind if rng.random() < 0.8 else ["f32", "f64", "i32"][int(rng.integers(0, 3))]
        packed = not (odd and rng.random() < 0.3)
        u = rng.random()
        extra = b""
        if odd and rng.random() < 0.3:
            extra = tag(15, 0) + varint(int(rng.integers(0, 1 << 40))) + ld(16, b"junk") + tag(17, 5) + b"\1\2\3\4"
        if u < 0.06:
            feats = [("other", value(kind, tensor(kind, _vals(rng, kind, width))))]
        elif u < 0.10:
            feats = [("values", value(raw=b"\x00\x01bytes"))]
        elif u < 0.13:
            feats = [("values", value())]
        else:
            sparse = mode == 1 or (mode == 2 and rng.random() < 0.5) or (mode == 3 and rng.random() < 0.4)
            w = width if rng.random() > 0.04 else width + 1
            if sparse and w > 0:
                k = int(rng.integers(1, w + 1))
                keys = rng.choice(w, k, replace=False)
                if rng.random() < 0.5:
                    keys = np.sort(keys)
                if rng.random() < 0.15:
                    keys = np.concatenate([keys, keys[:1]])               # a repeated key
                implicit = rng.random() < 0.3
                if implicit and w - 1 not in keys:
                    keys = np.concatenate([keys, [w - 1]])
                t = tensor(kind, _vals(rng, kind, len(keys)), keys, () if implicit else (w,), packed)
            else:
                t = tensor(kind, _vals(rng, kind, w), (), (w,) if rng.random() < 0.3 else (), packed)
            if odd and rng.random() < 0.2:
                t += tag(9, 0) + varint(5)                                 # an unknown field inside the tensor
            feats = [("values", value(kind, t))]
            if rng.random() < 0.2:
                feats.insert(0, ("aux", value("f64", tensor("f64", [1.0, 2.0]))))
        labs = []
        lu = rng.random()
        if lu < 0.75:
            lk = ["f32", "f64", "i32"][int(rng.integers(0, 3))]
            labs = [("values", value(lk, tensor(lk, _vals(rng, lk, 1 if rng.random() < 0.8 else int(rng.integers(0, 4))))))]
        elif lu < 0.85:
            labs = [("values", value(raw=b"x"))]
        recs.append(record(feats, labs, uid="r%d" % len(recs) if rng.random() < 0.3 else None, extra=extra))
    trailing = bytes(rng.integers(0, 256, int(rng.integers(1, 8)), dtype=np.uint8)) if rng.random() < 0.25 else b""
    return frame(recs, trailing)


def _uniform_body(parts, n):
    """n records whose payloads are the concatenation of `parts`: bytes (the same in every record) or (n, k) uint8 arrays."""
    cols = [np.frombuffer(p, np.uint8)[None, :].repeat(n, 0) if isinstance(p, bytes) else p for p in parts]
    L = sum(c.shape[1] for c in cols)
    head = np.frombuffer(struct.pack("<II", MAGIC, L), np.uint8)[None, :].repeat(n, 0)
    pad = np.zeros((n, -L % 4), np.uint8)
    return np.concatenate([head] + cols + [pad], axis=1).tobytes()


def big_dense_body(n, F, seed=0, kind="f32"):
    """n records of F float32 / float64 values each and one float32 label: (body, X float32, y float32) as numpy holds them."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, F)).astype(np.float32)
    X[rng.random((n, F)) < 0.01] = np.nan
    y = rng.integers(0, 2, n).astype(np.float32)
    xb = X.astype(np.float64 if kind == "f64" else np.float32)
    vbytes = xb.view(np.uint8).reshape(n, -1)
    t_head = tag(1, 2) + varint(vbytes.shape[1])
    v_head = tag(TENSOR_FIELD[kind], 2) + varint(len(t_head) + vbytes.shape[1])
    e_head = ld(1, b"values") + tag(2, 2) + varint(len(v_head) + len(t_head) + vbytes.shape[1])
    r_head = tag(1, 2) + varint(len(e_head) + len(v_head) + len(t_head) + vbytes.shape[1])
    lab = ld(1, b"values") + tag(2, 2) + varint(8) + tag(2, 2) + varint(6) + tag(1, 2) + varint(4)
    lab = tag(2, 2) + varint(len(lab) + 4) + lab
    body = _uniform_body([r_head + e_head + v_head + t_head, vbytes, lab, y.view(np.uint8).reshape(n, 4)], n)
    return body, X, y


def big_sparse_body(n, F, k, seed=0):
    """n sparse float32 records of width F (< 128) with exactly k entries each (sorted keys, shape [F]) and one label:
    (body, X with NaN = missing, y)."""
    assert F < 128
    rng = np.random.default_rng(seed)
    keys = np.sort(np.argsort(rng.random((n, F)), axis=1)[:, :k], axis=1).astype(np.uint8)
    vals = rng.standard_normal((n, k)).astype(np.float32)
    X = np.full((n, F), np.nan, np.float32)
    np.put_along_axis(X, keys.astype(np.int64), vals, axis=1)
    y = rng.standard_normal(n).astype(np.float32)
    tv, tk, ts = tag(1, 2) + varint(4 * k), tag(2, 2) + varint(k), ld(3, varint(F))
    tlen = len(tv) + 4 * k + len(tk) + k + len(ts)
    v_head = tag(2, 2) + varint(tlen)
    e_head = ld(1, b"values") + tag(2, 2) + varint(len(v_head) + tlen)
    r_head = tag(1, 2) + varint(len(e_head) + len(v_head) + tlen)
    lab = ld(1, b"values") + tag(2, 2) + varint(8) + tag(2, 2) + varint(6) + tag(1, 2) + varint(4)
    lab = tag(2, 2) + varint(len(lab) + 4) + lab
    body = _uniform_body([r_head + e_head + v_head + tv, vals.view(np.uint8).reshape(n, -1), tk, keys, ts + lab, y.view(np.uint8).reshape(n, 4)], n)
    return body, X, y


# ------------------------------------------------------------------------------------------------------------- the reference
def protobuf_available():
    try:
        import google.protobuf  # noqa: F401
        return True
    except ImportError:
        return False


def reference_available():
    return os.path.isfile(os.path.join(REFERENCE_SRC, "sagemaker_xgboost_container", "recordio_protobuf.py")) and protobuf_available()


def record_class():
    """aialgs.data.Record from descriptors (proto2, packed tensor fields)."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="b200_test_record.proto", package="aialgs.data", syntax="proto2")

    def add_field(msg, name, number, ftype, label=F.LABEL_OPTIONAL, type_name=None, packed=False, oneof=None):
        f = msg.field.add(name=name, number=number, type=ftype, label=label)
        if type_name:
            f.type_name = type_name
        if packed:
            f.options.packed = True
        if oneof is not None:
            f.oneof_index = oneof
    for name, t in (("Float32Tensor", F.TYPE_FLOAT), ("Float64Tensor", F.TYPE_DOUBLE), ("Int32Tensor", F.TYPE_INT32)):
        m = fd.message_type.add(name=name)
        add_field(m, "values", 1, t, F.LABEL_REPEATED, packed=True)
        add_field(m, "keys", 2, F.TYPE_UINT64, F.LABEL_REPEATED, packed=True)
        add_field(m, "shape", 3, F.TYPE_UINT64, F.LABEL_REPEATED, packed=True)
    b = fd.message_type.add(name="Bytes")
    add_field(b, "value", 1, F.TYPE_BYTES, F.LABEL_REPEATED)
    v = fd.message_type.add(name="Value")
    v.oneof_decl.add(name="value")
    add_field(v, "float32_tensor", 2, F.TYPE_MESSAGE, type_name=".aialgs.data.Float32Tensor", oneof=0)
    add_field(v, "float64_tensor", 3, F.TYPE_MESSAGE, type_name=".aialgs.data.Float64Tensor", oneof=0)
    add_field(v, "int32_tensor", 7, F.TYPE_MESSAGE, type_name=".aialgs.data.Int32Tensor", oneof=0)
    add_field(v, "bytes", 9, F.TYPE_MESSAGE, type_name=".aialgs.data.Bytes", oneof=0)
    r = fd.message_type.add(name="Record")
    for name, number in (("features", 1), ("label", 2)):
        entry = r.nested_type.add(name=name.capitalize() + "Entry")
        entry.options.map_entry = True
        add_field(entry, "key", 1, F.TYPE_STRING)
        add_field(entry, "value", 2, F.TYPE_MESSAGE, type_name=".aialgs.data.Value")
        add_field(r, name, number, F.TYPE_MESSAGE, F.LABEL_REPEATED, type_name=".aialgs.data.Record.%sEntry" % name.capitalize())
    for name, number in (("uid", 3), ("metadata", 4), ("configuration", 5)):
        add_field(r, name, number, F.TYPE_STRING)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("aialgs.data.Record"))


def reference_reader():
    """The reference's read_recordio_protobuf, with sagemaker_containers.record_pb2 stubbed by record_class()."""
    Record = record_class()
    saved = {k: sys.modules.get(k) for k in ("sagemaker_containers", "sagemaker_containers.record_pb2")}
    pkg = types.ModuleType("sagemaker_containers")
    pb2 = types.ModuleType("sagemaker_containers.record_pb2")
    pb2.Record = Record
    pkg.record_pb2 = pb2
    sys.modules["sagemaker_containers"], sys.modules["sagemaker_containers.record_pb2"] = pkg, pb2
    try:
        spec = importlib.util.spec_from_file_location("_reference_recordio_protobuf", os.path.join(REFERENCE_SRC, "sagemaker_xgboost_container", "recordio_protobuf.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    return mod.read_recordio_protobuf, Record
