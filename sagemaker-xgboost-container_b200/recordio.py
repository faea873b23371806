"""recordio-protobuf (application/x-recordio-protobuf) bodies -> DMatrix.

The container decodes these with `read_recordio_protobuf` (recordio_protobuf.py, on `sagemaker_containers.record_pb2`) and
builds `xgb.DMatrix(features, label=labels)`.  Here the body goes to the device as it is and is decoded there
(XGB200DMatrixCreateFromRecordIO, csrc/recordio.cu).  The few bodies the device path hands back (status 2: unpacked or repeated
fields, merged messages, a repeated "values" key, malformed protobuf ...) are decoded by `read_recordio_protobuf` below, a
wire-format walker in plain Python that follows protobuf's parsing rules and the reference's row rules (DESIGN.md
"recordio-protobuf"); it needs neither record_pb2 nor google.protobuf.
"""
import struct

import numpy as np

from .backend import get_backend

_MAGIC = 0xCED7230A
_F32, _F64, _I32, _BYTES = 2, 3, 7, 9                # Value oneof: float32_tensor, float64_tensor, int32_tensor, bytes
_U64 = (1 << 64) - 1


class DecodeError(ValueError):
    """A record that is not a valid protobuf message."""


def _records(buf):
    """(start, stop) of each record's payload; the framing rules of the container's reader."""
    offset, n = 0, len(buf)
    while offset + 8 <= n:                           # 1 to 7 trailing bytes are ignored
        magic, length = struct.unpack_from("<II", buf, offset)
        if magic != _MAGIC:
            raise ValueError(f"Invalid RecordIO magic at offset {offset}")
        offset += 8
        padded = (length + 3) // 4 * 4
        if offset + padded > n:
            raise ValueError(f"Truncated record at offset {offset}")
        yield offset, offset + length
        offset += padded


def _varint(buf, pos, end):
    result, shift = 0, 0
    while True:
        if pos >= end:
            raise DecodeError("Truncated varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result & _U64, pos
        shift += 7
        if shift >= 70:
            raise DecodeError("Too many bytes when decoding varint")


def _fields(buf, pos, end):
    """(field number, wire type, value) of a message: the int of a varint, else the (start, stop) of the field's bytes."""
    while pos < end:
        tag, pos = _varint(buf, pos, end)
        fnum, wt = tag >> 3, tag & 7
        if fnum == 0 or tag > 0xFFFFFFFF:
            raise DecodeError("Invalid tag")
        if wt == 0:
            v, pos = _varint(buf, pos, end)
        elif wt in (1, 5):
            size = 8 if wt == 1 else 4
            if pos + size > end:
                raise DecodeError("Truncated fixed-size field")
            v, pos = (pos, pos + size), pos + size
        elif wt == 2:
            size, pos = _varint(buf, pos, end)
            if pos + size > end:
                raise DecodeError("Truncated length-delimited field")
            v, pos = (pos, pos + size), pos + size
        else:
            raise DecodeError("Unsupported wire type %d" % wt)
        yield fnum, wt, v


def _packed_varints(buf, start, stop):
    out, pos = [], start
    while pos < stop:
        v, pos = _varint(buf, pos, stop)
        out.append(v)
    return out


def _as_int32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v & 0x80000000 else v


def _tensor(buf, case):
    """A tensor message -> (values, keys or None, shape or None), the arrays the container's reader builds."""
    vals, keys, shape = [], [], []
    scalar_wt = {_F32: 5, _F64: 1, _I32: 0}[case]
    for fnum, wt, v in _fields(buf, 0, len(buf)):
        if fnum == 1 and wt == 2:                     # packed values
            chunk = bytes(buf[v[0]:v[1]])
            if case == _I32:
                vals.extend(_as_int32(x) for x in _packed_varints(buf, v[0], v[1]))
            else:
                size = 4 if case == _F32 else 8
                if len(chunk) % size:
                    raise DecodeError("Packed fixed-size field of a wrong length")
                vals.append(np.frombuffer(chunk, "<f4" if case == _F32 else "<f8"))
        elif fnum == 1 and wt == scalar_wt:           # unpacked values
            if case == _I32:
                vals.append(_as_int32(v))
            else:
                vals.append(np.frombuffer(bytes(buf[v[0]:v[1]]), "<f4" if case == _F32 else "<f8"))
        elif fnum in (2, 3) and wt in (0, 2):         # keys / shape, packed or not
            dst = keys if fnum == 2 else shape
            dst.extend(_packed_varints(buf, v[0], v[1]) if wt == 2 else [v])
        # anything else is an unknown field (a known field with another wire type included): skipped
    if case == _I32:
        values = np.array(vals, dtype=np.int32)
    else:
        parts = [np.atleast_1d(p) for p in vals]
        values = np.concatenate(parts) if parts else np.zeros(0, "<f4" if case == _F32 else "<f8")
        # protobuf hands float32 values to Python as doubles: a signalling NaN comes back quiet
        values = values.astype(np.float64).astype(np.float32) if case == _F32 else values.astype(np.float64)
    return values, (np.array(keys, dtype=np.uint64) if keys else None), (shape if shape else None)


def _value(buf):
    """A Value message -> (values, keys, shape) of its tensor, or None when it holds none (bytes, or nothing set)."""
    case, parts = None, []
    for fnum, wt, v in _fields(buf, 0, len(buf)):
        if wt != 2 or fnum not in (_F32, _F64, _I32, _BYTES):
            continue
        if fnum != case:                              # another oneof member replaces the one set before
            parts = []
        case = fnum
        parts.append(bytes(buf[v[0]:v[1]]))           # the same member again merges (= parsing the concatenation)
    if case in (_F32, _F64, _I32):
        return _tensor(b"".join(parts), case)
    return None


def _record(buf, start, stop):
    """A Record -> ({key: Value} of features, of label); every Value is parsed, as protobuf does."""
    maps = {1: {}, 2: {}}
    for fnum, wt, v in _fields(buf, start, stop):
        if fnum not in (1, 2) or wt != 2:
            continue                                  # uid / metadata / configuration and unknown fields
        key, parts = b"", []
        for efnum, ewt, ev in _fields(buf, v[0], v[1]):
            if ewt != 2:
                continue
            if efnum == 1:
                key = bytes(buf[ev[0]:ev[1]])
            elif efnum == 2:
                parts.append(bytes(buf[ev[0]:ev[1]]))
        maps[fnum][key] = _value(b"".join(parts))     # a key given again replaces the entry
    return maps[1], maps[2]


def read_recordio_protobuf(buf):
    """recordio-protobuf bytes -> (features: ndarray or scipy CSR, labels: ndarray or None), with the container's rules:
    features["values"] of each record is a row -- sparse when its tensor has keys (width shape[0], else max key + 1), dense
    otherwise; a record without it, or whose Value holds no tensor, is skipped with its label; one sparse row makes the whole
    batch sparse (scipy.sparse.vstack), else np.vstack; labels are every kept record's label["values"] values."""
    from scipy.sparse import csr_matrix, vstack
    buf = memoryview(buf).cast("B")
    rows, labels, sparse = [], [], False
    for start, stop in _records(buf):
        features, label = _record(buf, start, stop)
        tensor = features.get(b"values")
        if tensor is None:
            continue
        values, keys, shape = tensor
        if keys is not None:
            sparse = True
            ncols = int(shape[0]) if shape else int(keys.max()) + 1
            rows.append(csr_matrix((values, keys.astype(np.int64), [0, len(keys)]), shape=(1, ncols)))
        else:
            rows.append(values.reshape(1, -1))
        lab = label.get(b"values")
        if lab is not None:
            labels.append(lab[0])
    if not rows:
        raise ValueError("No records found in RecordIO-Protobuf data")
    features = vstack(rows).tocsr() if sparse else np.vstack(rows)
    return features, (np.concatenate(labels, axis=None) if labels else None)


def recordio_protobuf_to_dmatrix(buf):
    """recordio-protobuf bytes (bytes, bytearray, memoryview) -> DMatrix: decoded on the device; bodies the device path hands
    back are decoded by read_recordio_protobuf; a body the container's reader rejects raises ValueError."""
    from .core import DMatrix
    be = get_backend()
    if hasattr(be, "dmatrix_from_recordio"):
        handle, status, message = be.dmatrix_from_recordio(buf)
        if status == 0:
            return DMatrix._from_handle(handle)
        if status == 1:
            raise ValueError(message)
    features, labels = read_recordio_protobuf(buf)
    return DMatrix(features, label=labels)
