"""Text loaders behind `DMatrix("<path>?format=csv&label_column=0&delimiter=,")` and `?format=libsvm`.

The container builds these URIs at data_utils.py:309-313 (CSV, optional weight_column=1) and :361 (libsvm) and
points them at a directory of symlinks (data_utils.py:520-545, 624-628): every regular file in it is loaded.
Upstream parses with dmlc-core's multi-threaded text parsers; here pandas' C parser does the CSV and a small
vectorised tokenizer the libsvm text.  Feature indices of libsvm files are kept as-is (abalone's 1-based
indices give 9 columns, test/unit/test_data_utils.py:119-127).
"""
import os
from urllib.parse import parse_qs

import numpy as np

from .backend import XGBoostError


def _list_files(path):
    if os.path.isdir(path):
        files = sorted(os.path.join(path, f) for f in os.listdir(path) if os.path.isfile(os.path.join(path, f)))
        if not files:
            raise XGBoostError("No files found in %s" % path)
        return files
    if os.path.isfile(path):
        return [path]
    raise XGBoostError("Opening %s failed: No such file or directory" % path)


def parse_uri(uri):
    path, _, query = uri.partition("?")
    q = {k: v[0] for k, v in parse_qs(query, keep_blank_values=True).items()}
    # `delimiter=,` style values survive parse_qs unchanged; a literal '&'/'#' delimiter is not expressible upstream either
    return path, q


def _load_csv(files, q):
    import pandas as pd
    delim = q.get("delimiter", ",")
    label_col = int(q["label_column"]) if "label_column" in q else None
    weight_col = int(q["weight_column"]) if "weight_column" in q else None
    frames = []
    for f in files:
        if os.path.getsize(f) == 0:
            continue
        try:
            df = pd.read_csv(f, header=None, sep=delim, dtype=np.float32, na_values=["", "nan", "NaN", "NA"], keep_default_na=True,
                             engine="c", skip_blank_lines=True)
        except Exception as e:
            raise XGBoostError("Failed to parse CSV file %s: %s" % (f, e))
        frames.append(df.to_numpy(dtype=np.float32, copy=False))
    if not frames:
        raise XGBoostError("CSV input is empty")
    ncol = {a.shape[1] for a in frames}
    if len(ncol) != 1:
        raise XGBoostError("CSV files have different numbers of columns: %s" % sorted(ncol))
    data = np.concatenate(frames, axis=0) if len(frames) > 1 else frames[0]
    y = w = None
    drop = []
    if label_col is not None:
        y = np.ascontiguousarray(data[:, label_col])
        drop.append(label_col)
    if weight_col is not None:
        w = np.ascontiguousarray(data[:, weight_col])
        drop.append(weight_col)
    if drop:
        keep = [c for c in range(data.shape[1]) if c not in drop]
        data = np.ascontiguousarray(data[:, keep])
    return data, y, w


def _has_qid(fh, chunk=1 << 22):
    """Whether the rest of the file holds a `qid:` token, read in fixed-size chunks (a token split by a chunk edge is kept whole by
    carrying the last three bytes over)."""
    tail = b""
    while True:
        block = fh.read(chunk)
        if not block:
            return False
        if b"qid:" in tail + block[:3] or b"qid:" in block:
            return True
        tail = block[-3:]


def _load_libsvm_fast(files):
    """C parser of scikit-learn when the files are plain `label idx:val ...` lines (no per-row weights / qid: that parser would
    drop a qid token on any line, so a file with one anywhere goes to the plain loop)."""
    try:
        from sklearn.datasets import load_svmlight_files
    except ImportError:
        return None
    for f in files:
        with open(f, "rb") as fh:
            head = fh.readline().split(b"#", 1)[0].split()
            if not head or b":" in head[0] or _has_qid(fh):
                return None
        if any(t.startswith(b"qid:") for t in head[1:]):
            return None
    try:
        out = load_svmlight_files(files, dtype=np.float32, zero_based=True)
    except Exception:
        return None
    import scipy.sparse as sp
    Xs, ys = out[0::2], out[1::2]
    ncol = max(x.shape[1] for x in Xs)
    Xs = [sp.csr_matrix((x.data, x.indices, x.indptr), shape=(x.shape[0], ncol)) for x in Xs]
    X = sp.vstack(Xs, format="csr") if len(Xs) > 1 else Xs[0]
    return X, np.concatenate(ys).astype(np.float32), None


def _load_libsvm(files, q, with_qid=False):
    """-> (CSR features, labels, weights | None), plus the qid of every row (int64, or None without qid tokens) with with_qid.
    A file with qid tokens must carry one on every line; the query groups are the runs of equal consecutive qid."""
    import scipy.sparse as sp
    fast = _load_libsvm_fast(files)
    if fast is not None:
        return fast + (None,) if with_qid else fast
    labels, weights, rows_ptr, cols, vals, qids = [], [], [0], [], [], []
    has_weight = False
    for f in files:
        with open(f, "rb") as fh:
            for line in fh:
                line = line.split(b"#", 1)[0].strip()
                if not line:
                    continue
                parts = line.split()
                head = parts[0]
                if b":" in head:
                    lab, wt = head.split(b":", 1)
                    labels.append(float(lab))
                    weights.append(float(wt))
                    has_weight = True
                else:
                    labels.append(float(head))
                    weights.append(1.0)
                for tok in parts[1:]:
                    k, _, v = tok.partition(b":")
                    if k == b"qid":
                        if len(qids) >= len(labels):
                            raise XGBoostError("Invalid libsvm token %r in %s: a second qid on the line" % (tok, f))
                        try:
                            qids.extend([None] * (len(labels) - 1 - len(qids)) + [int(v)])
                        except ValueError:
                            raise XGBoostError("Invalid libsvm token %r in %s" % (tok, f))
                        continue
                    try:
                        cols.append(int(k))
                        vals.append(float(v))
                    except ValueError:
                        raise XGBoostError("Invalid libsvm token %r in %s" % (tok, f))
                rows_ptr.append(len(cols))
    if not labels:
        raise XGBoostError("libsvm input is empty")
    ncol = (max(cols) + 1) if cols else 0
    X = sp.csr_matrix((np.asarray(vals, np.float32), np.asarray(cols, np.int32), np.asarray(rows_ptr, np.int64)), shape=(len(labels), ncol))
    out = (X, np.asarray(labels, np.float32), (np.asarray(weights, np.float32) if has_weight else None))
    n_qid = sum(1 for x in qids if x is not None)
    if n_qid and n_qid != len(labels):
        raise XGBoostError("libsvm input: %d of %d rows have a qid token; all or none must" % (n_qid, len(labels)))
    return out + (np.asarray(qids, np.int64) if n_qid else None,) if with_qid else out


def load_uri(uri, with_qid=False):
    """-> (features: ndarray | scipy CSR, label | None, weight | None), plus the per-row qid of a libsvm input (None without qid
    tokens, and for CSV) with with_qid"""
    path, q = parse_uri(uri)
    fmt = q.get("format")
    if fmt is None:
        ext = os.path.splitext(path)[1].lower()
        fmt = "csv" if ext == ".csv" else "libsvm"
    files = _list_files(path)
    if fmt == "csv":
        out = _load_csv(files, q)
        return out + (None,) if with_qid else out
    if fmt == "libsvm":
        return _load_libsvm(files, q, with_qid)
    raise XGBoostError("Unknown data format in URI: %s" % fmt)


def _arrow_columns(table):
    """pyarrow Table -> one numpy array per column without assembling a frame: a column without nulls is handed over in its
    own dtype (zero-copy for a single chunk), nulls become NaN (float64, as Table.to_pandas does for numeric columns)."""
    cols = []
    for i in range(table.num_columns):
        col = table.column(i)
        if col.num_chunks != 1:
            col = col.combine_chunks()
        else:
            col = col.chunk(0)
        try:
            cols.append(col.to_numpy(zero_copy_only=col.null_count == 0))
        except Exception:
            cols.append(np.asarray(col.to_numpy(zero_copy_only=False), np.float32))
    return cols


def _is_data_file(file_path, file_name):
    """data_utils._is_data_file (data_utils.py:120-139): a regular file, not hidden, not an xgboost cache file."""
    if not os.path.isfile(os.path.join(file_path, file_name)):
        return False
    if file_name.startswith(".") or file_name.startswith("_"):
        return False
    return not (".cache" in file_name and ("dtrain" in file_name or "dval" in file_name))


def recordio_protobuf_to_dmatrix(files_path, is_pipe=False):
    """recordio-protobuf channel -> DMatrix, or None when the directory holds no data file: what
    data_utils.get_recordio_protobuf_dmatrix builds (data_utils.py:418-459).  The files, sorted, are read into one buffer
    (no second copy to join them) that is decoded on the device (csrc/recordio.cu).  Pipe mode is refused, as there."""
    if is_pipe:
        raise XGBoostError("Pipe mode for RecordIO-Protobuf is no longer supported. Please use Fast File mode (default) instead. "
                           "Set input_mode='File' in your SageMaker Estimator or TrainingInput.")
    from .recordio import recordio_protobuf_to_dmatrix as to_dmatrix
    if os.path.isfile(files_path):
        paths = [files_path]
    else:
        paths = [os.path.join(files_path, f) for f in sorted(os.listdir(files_path)) if _is_data_file(files_path, f)]
    if not paths:
        return None
    sizes = [os.path.getsize(p) for p in paths]
    buf = bytearray(sum(sizes))
    view, at = memoryview(buf), 0
    for p, size in zip(paths, sizes):
        with open(p, "rb") as fh:
            got = fh.readinto(view[at:at + size])
        if got != size:
            raise XGBoostError("%s changed size while it was read" % p)
        at += size
    return to_dmatrix(buf)


def parquet_to_dmatrix(files_path):
    """Parquet channel -> DMatrix, column 0 = label (what data_utils._get_parquet_dmatrix_file_mode builds, data_utils.py:368-390)
    without its host copies (Table -> DataFrame -> ndarray -> data[:, 1:]): the arrow column buffers go to the device as they are
    and are converted / transposed there (csrc/ingest.cu).  Optional binding in the container, like encoder.csv_to_dmatrix:

        def _get_parquet_dmatrix_file_mode(files_path):
            return sagemaker_xgboost_container_b200.data.parquet_to_dmatrix(files_path)
    """
    import pyarrow.parquet as pq
    from .backend import get_backend
    from .core import DMatrix
    table = pq.read_table(files_path)
    be = get_backend()
    if table.num_columns < 1:
        raise XGBoostError("Parquet input has no columns")
    if not hasattr(be, "dmatrix_from_columns"):
        data = table.to_pandas().to_numpy()
        return DMatrix(data[:, 1:], label=data[:, 0])
    return DMatrix._from_handle(be.dmatrix_from_columns(_arrow_columns(table), label_column=0))
