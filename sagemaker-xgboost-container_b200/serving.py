"""Serving input path of the container on the device (SURVEY.md section 8f row 1; BASELINE config 5).

Mirrors, with the same names / arguments / error behaviour, the two reference functions a `text/csv` invocation goes through:

    encoder.csv_to_dmatrix(input, dtype=None)                              encoder.py:35-52
    serve_utils.predict(model, model_format, dtest, input_content_type,   algorithm_mode/serve_utils.py:200-262
                        objective=None)

`csv_to_dmatrix` hands the request body to the engine, which parses it on the GPU straight into the DMatrix
(XGB200DMatrixCreateFromCSV, csrc/csv.cu) instead of `str.split` + `np.array(...).astype(float)` on the host; bodies the exact
device fast path cannot decide (e.g. 30-digit literals) take the reference's own host route, so values never differ.
`predict` is the container's single-model / ensemble logic over `Booster.predict`.  INTEGRATION.md shows the two-line change
in encoder.py that routes the container through this module.
"""
import csv
import logging

import numpy as np

from .backend import XGBoostError, get_backend
from .core import Booster, DMatrix

MULTI_SOFTMAX = "multi:softmax"        # constants/xgb_constants.py
BINARY_HINGE = "binary:hinge"


def _sniff_delimiter(first_line):
    sniffed = csv.Sniffer().sniff(first_line[:512]).delimiter          # encoder.py:46-47
    return "," if sniffed.isalnum() else sniffed


def _host_csv_to_array(csv_string, delimiter, dtype):
    """The reference's own route (encoder.py:31-32,50)."""
    rows = [["nan" if x == "" else x for x in line.split(delimiter)] for line in csv_string.split("\n")]
    return np.array(rows).astype(dtype)


def csv_to_dmatrix(input, dtype=None):
    """Convert a CSV object (str, or bytes encoded as UTF-8, already stripped of leading / trailing newlines) to a DMatrix."""
    # no copy of a 200 MB body on the way in: the first line is sliced out (str.split(..., 1) would copy the remainder) and a
    # str payload is handed to the library through its cached UTF-8 buffer (backend.dmatrix_from_csv)
    end = input.find("\n" if isinstance(input, str) else b"\n")
    first = input[:end] if end >= 0 else input
    delimiter = _sniff_delimiter(first if isinstance(first, str) else first.decode("utf-8"))
    logging.info("Determined delimiter of CSV input is '{}'".format(delimiter))
    be = get_backend()
    if len(delimiter) == 1 and ord(delimiter) < 128 and hasattr(be, "dmatrix_from_csv"):
        handle, status = be.dmatrix_from_csv(input, delimiter)
        if status == 0:
            return DMatrix._from_handle(handle)
        if status == 1:          # numpy raises on ragged rows as well (inhomogeneous shape)
            raise ValueError("setting an array element with a sequence. The requested array has an inhomogeneous shape: rows of the CSV payload have different numbers of fields")
    return DMatrix(_host_csv_to_array(input if isinstance(input, str) else input.decode("utf-8"), delimiter, float if dtype is None else dtype))


def _host_sparse_matrix_from_libsvm(payload):
    """The reference's own route (algorithm_mode/serve_utils.py:94-118), kept for the bodies the device parser hands back."""
    from scipy.sparse import csr_matrix
    row, col, data = [], [], []
    for row_idx, line in enumerate(x.split(" ") for x in payload.split("\n")):
        for item in line:
            if ":" in item:
                parts = item.split(":")
                col.append(int(parts[0]))
                row.append(row_idx)
                data.append(parts[1])
    row, col = np.array(row), np.array(col).astype(int)
    if len(col) > 0 and col.min() >= 1:
        col = col - 1
    data = np.array(data).astype(float)
    if not (len(row) == len(col) and len(col) == len(data)):
        raise RuntimeError("Dimension checking failed when transforming sparse matrix.")
    return csr_matrix((data, (row, col)))


def sparse_libsvm_to_dmatrix(payload):
    """`xgb.DMatrix(_get_sparse_matrix_from_libsvm(decoded_payload))` of serve_utils.parse_content_data (serve_utils.py:132-137)
    in one step: the body (str, already stripped) is parsed on the device, entries a line does not list are missing."""
    be = get_backend()
    if hasattr(be, "dmatrix_from_libsvm_text") and len(payload) > 0:
        handle, status = be.dmatrix_from_libsvm_text(payload, 0, float("nan"))
        if status == 0:
            return DMatrix._from_handle(handle)
    return DMatrix(_host_sparse_matrix_from_libsvm(payload if isinstance(payload, str) else payload.decode("utf-8")))


def _host_libsvm_rows(string_like):
    rows = []
    for line in string_like.strip().split("\n"):                 # encoder.py:64-72
        row = {}
        for token in line.strip().split():
            if ":" in token:
                idx, val = token.split(":", 1)
                row[int(idx)] = float(val)
        rows.append(row)
    return rows


def libsvm_to_dmatrix(string_like):
    """encoder.libsvm_to_dmatrix (encoder.py:54-86): dense matrix, entries a line does not list are 0.0."""
    if isinstance(string_like, (bytes, bytearray)):
        string_like = string_like.decode("utf-8")
    body = string_like.strip()
    be = get_backend()
    if hasattr(be, "dmatrix_from_libsvm_text") and len(body) > 0:
        handle, status = be.dmatrix_from_libsvm_text(body, 1, 0.0)
        if status == 0:
            return DMatrix._from_handle(handle)
    rows = _host_libsvm_rows(string_like)
    if not rows or not any(rows):
        return DMatrix(np.empty((0, 0)))
    min_idx = min(idx for row in rows for idx in row)
    offset = 1 if min_idx >= 1 else 0
    max_col = max(idx for row in rows for idx in row) - offset + 1
    data = np.zeros((len(rows), max_col))
    for i, row in enumerate(rows):
        for idx, val in row.items():
            data[i, idx - offset] = val
    return DMatrix(data)


def recordio_protobuf_to_dmatrix(string_like):
    """encoder.recordio_protobuf_to_dmatrix (encoder.py:90-99): a recordio-protobuf request body (bytes-like) -> DMatrix,
    decoded on the device (csrc/recordio.cu); bodies the device path hands back take the package's host walker."""
    from .recordio import recordio_protobuf_to_dmatrix as to_dmatrix
    return to_dmatrix(string_like)


def _predict_one(booster, dtest):
    best_iteration = getattr(booster, "best_ntree_limit", 0)          # serve_utils.py:228-250
    try:
        best_iteration = int(best_iteration) if best_iteration is not None else 0
    except (TypeError, ValueError):
        best_iteration = 0
    if best_iteration > 0:
        return booster.predict(dtest, iteration_range=(0, best_iteration), validate_features=False)
    return booster.predict(dtest, validate_features=False)


def predict(model, model_format, dtest, input_content_type, objective=None):
    """Single model: Booster.predict.  List of models: vote (multi:softmax / binary:hinge) or mean of the members."""
    if isinstance(model, list):
        ensemble = [_predict_one(b, dtest) for b in model]
        if objective in (MULTI_SOFTMAX, BINARY_HINGE):
            from scipy import stats
            return stats.mode(ensemble).mode[0]
        return np.mean(ensemble, axis=0)
    return _predict_one(model, dtest)


__all__ = ["csv_to_dmatrix", "sparse_libsvm_to_dmatrix", "libsvm_to_dmatrix", "recordio_protobuf_to_dmatrix", "predict", "Booster", "DMatrix", "XGBoostError"]
