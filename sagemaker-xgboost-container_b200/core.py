"""DMatrix / Booster with the surface of `xgboost.core` that the SageMaker container consumes.

Reference call sites (aws/sagemaker-xgboost-container, under src/sagemaker_xgboost_container):
  DMatrix   data_utils.py:309-313,361,384,453,586  encoder.py:52,76,87,98  serve_utils.py:137,205  train.py:339-342,394-411
  Booster   serve_utils.py:180-250  serve.py:85-88  serving.py:98  train.py:445,480-485  checkpointing.py:375,428
Semantics follow upstream python-package/xgboost/core.py @ v3.0.5 (SURVEY.md Appendix A).
"""
import json
import os
import warnings

import numpy as np

from .backend import XGBoostError, get_backend  # noqa: F401  (re-exported like xgboost.core)
from .data import load_uri


def _is_scipy_sparse(x):
    try:
        import scipy.sparse as sp
        return sp.issparse(x)
    except ImportError:  # pragma: no cover
        return False


def _is_pandas_df(x):
    return type(x).__module__.startswith("pandas") and hasattr(x, "columns") and hasattr(x, "to_numpy")


class DMatrix:
    """Data matrix resident on the GPU (raw float32 features; the binned feature blocks are built on first training use)."""

    def __init__(self, data, label=None, *, weight=None, base_margin=None, missing=None, silent=False, feature_names=None,
                 feature_types=None, nthread=None, group=None, qid=None, label_lower_bound=None, label_upper_bound=None,
                 feature_weights=None, enable_categorical=False, data_split_mode=None):
        self.handle = None
        if isinstance(data, DataIter):
            raise XGBoostError("DMatrix(DataIter) (external memory) is not supported by the CUDA hist path; build a QuantileDMatrix from the "
                               "iterator instead")
        if group is not None or qid is not None:
            _check_ranking_backend()
        if enable_categorical:
            raise XGBoostError("categorical features are not supported on the CUDA hist path")
        be = get_backend()
        miss = np.nan if missing is None else float(missing)
        if isinstance(data, (str, os.PathLike)) and self._try_device_csv(os.fspath(data), be):
            pass
        elif isinstance(data, (str, os.PathLike)):
            X, y, w, q = load_uri(os.fspath(data), with_qid=True)
            if q is not None and qid is None and group is None:
                _check_ranking_backend()
                qid = q
            if _is_scipy_sparse(X):
                self.handle = be.dmatrix_from_csr(X.indptr, X.indices, X.data, X.shape[1])
            else:
                self.handle = be.dmatrix_from_dense(X, np.nan)
            if label is None and y is not None:
                label = y
            if weight is None and w is not None:
                weight = w
        elif hasattr(data, "__cuda_array_interface__"):
            self.handle = be.dmatrix_from_cuda_array(data, missing)
        elif _is_scipy_sparse(data):
            csr = data.tocsr()
            self.handle = be.dmatrix_from_csr(csr.indptr, csr.indices, csr.data, csr.shape[1])
        elif _is_pandas_df(data):
            if feature_names is None:
                feature_names = [str(c) for c in data.columns]
            if hasattr(be, "dmatrix_from_columns") and missing is None and len(data.columns) > 0 and all(
                    isinstance(t, np.dtype) and t.kind in "fiub" for t in data.dtypes):
                # column buffers straight to the device (csrc/ingest.cu): no dense float32 copy of the frame on the host
                self.handle = be.dmatrix_from_columns([data.iloc[:, j].to_numpy() for j in range(len(data.columns))])
            else:
                self.handle = be.dmatrix_from_dense(data.to_numpy(dtype=np.float32, na_value=np.nan) if hasattr(data, "to_numpy") else np.asarray(data), miss)
        elif isinstance(data, DMatrix):
            raise TypeError("cannot construct a DMatrix from a DMatrix")
        else:
            arr = np.asarray(data)
            if arr.dtype == object:
                arr = arr.astype(np.float32)
            if arr.ndim == 1:
                arr = arr.reshape(-1, 1)
            if arr.ndim != 2:
                raise ValueError("Expecting 2 dimensional numpy.ndarray, got: %s" % (arr.shape,))
            self.handle = be.dmatrix_from_dense(arr, miss)
        if label is not None:
            self.set_label(label)
        if weight is not None:
            self.set_weight(weight)
        if base_margin is not None:
            self.set_base_margin(base_margin)
        if label_lower_bound is not None:
            self.set_float_info("label_lower_bound", label_lower_bound)
        if label_upper_bound is not None:
            self.set_float_info("label_upper_bound", label_upper_bound)
        if group is not None:
            self.set_group(group)
        if qid is not None:
            self.set_info(qid=qid)
        if feature_names is not None:
            self.feature_names = feature_names
        if feature_types is not None:
            self.feature_types = feature_types

    def _try_device_csv(self, uri, be):
        """CSV channels go to the device as TEXT and are parsed there (csrc/csv.cu) -- no dense float32 host copy.  Returns
        False (host loader takes over) for other formats, backends without the entry point, or text the exact device fast
        path cannot decide (blank lines inside a file, >19-digit literals, ragged rows: the host loader reports those)."""
        from .data import parse_uri, _list_files
        if not hasattr(be, "dmatrix_from_csv_labeled"):
            return False
        path, q = parse_uri(uri)
        fmt = q.get("format") or ("csv" if os.path.splitext(path)[1].lower() == ".csv" else "libsvm")
        delim = q.get("delimiter", ",")
        if fmt != "csv" or len(delim) != 1 or ord(delim) >= 128:
            return False
        chunks = []
        for f in _list_files(path):
            with open(f, "rb") as fh:
                b = fh.read().strip()
            if b:
                chunks.append(b.replace(b"\r\n", b"\n"))
        if not chunks:
            return False
        handle, status = be.dmatrix_from_csv_labeled(b"\n".join(chunks), delim, int(q.get("label_column", -1)), int(q.get("weight_column", -1)))
        if status != 0:
            return False
        self.handle = handle
        return True

    @classmethod
    def _from_handle(cls, handle):
        obj = cls.__new__(cls)
        obj.handle = handle
        return obj

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None:
            try:
                get_backend().dmatrix_free(h)
            except Exception:  # pragma: no cover - interpreter shutdown
                pass
            self.handle = None

    # NB: no __len__/__bool__: the container uses DMatrix objects in boolean context (train.py:243,271).
    def num_row(self):
        return get_backend().dmatrix_num_row(self.handle)

    def num_col(self):
        return get_backend().dmatrix_num_col(self.handle)

    def set_float_info(self, field, data):
        get_backend().dmatrix_set_float_info(self.handle, field, np.asarray(data, dtype=np.float32))

    def get_float_info(self, field):
        return get_backend().dmatrix_get_float_info(self.handle, field)

    def set_label(self, label):
        """A 1-D label, or an (n, T) numpy / pandas one for multi-target regression (T label columns); an (n, 1) label is the 1-D
        label.  get_label() returns the labels flat, row-major."""
        a = label.to_numpy(dtype=np.float32, na_value=np.nan) if _is_pandas_df(label) else np.asarray(label, dtype=np.float32)
        if a.ndim == 2 and a.shape[1] > 1:
            get_backend().dmatrix_set_info_interface(self.handle, "label", np.ascontiguousarray(a))
        else:
            self.set_float_info("label", a)

    def set_weight(self, weight):
        self.set_float_info("weight", weight)

    def set_base_margin(self, margin):
        self.set_float_info("base_margin", margin)

    def get_label(self):
        return self.get_float_info("label")

    def get_weight(self):
        return self.get_float_info("weight")

    def get_base_margin(self):
        return self.get_float_info("base_margin")

    # ---- query groups (rank:* objectives, ndcg / map metrics); under groups a weight is one per group
    def set_group(self, group):
        _check_ranking_backend()
        get_backend().dmatrix_set_group(self.handle, np.asarray(group, dtype=np.uint32))

    def set_uint_info(self, field, data):
        _check_ranking_backend()
        get_backend().dmatrix_set_uint_info(self.handle, field, np.asarray(data, dtype=np.uint32))

    def get_uint_info(self, field):
        be = get_backend()
        return be.dmatrix_get_uint_info(self.handle, field) if getattr(be, "supports_ranking", False) else np.zeros(0, np.uint32)

    def get_group(self):
        ptr = self.get_uint_info("group_ptr")
        return np.diff(ptr).astype(np.uint32) if len(ptr) else np.zeros(0, np.uint32)

    def set_info(self, *, label=None, weight=None, base_margin=None, label_lower_bound=None, label_upper_bound=None, feature_names=None,
                 feature_types=None, group=None, qid=None, **kwargs):
        if group is not None:
            self.set_group(group)
        if qid is not None:
            _check_ranking_backend()
            q = np.asarray(qid)
            get_backend().dmatrix_set_info_interface(self.handle, "qid", q if q.dtype.kind in "iu" else q.astype(np.float64))
        if label is not None:
            self.set_label(label)
        if weight is not None:
            self.set_weight(weight)
        if base_margin is not None:
            self.set_base_margin(base_margin)
        if label_lower_bound is not None:
            self.set_float_info("label_lower_bound", label_lower_bound)
        if label_upper_bound is not None:
            self.set_float_info("label_upper_bound", label_upper_bound)
        if feature_names is not None:
            self.feature_names = feature_names
        if feature_types is not None:
            self.feature_types = feature_types
        for k, v in kwargs.items():
            if v is not None:
                raise XGBoostError("DMatrix.set_info: field %r is not supported on the CUDA hist path" % k)

    def slice(self, rindex, allow_groups=False):
        idx = np.asarray(list(rindex) if not isinstance(rindex, np.ndarray) else rindex, dtype=np.int32)
        be = get_backend()
        h = be.dmatrix_slice(self.handle, idx, allow_groups=True) if allow_groups else be.dmatrix_slice(self.handle, idx)
        return DMatrix._from_handle(h)

    @property
    def feature_names(self):
        v = get_backend().dmatrix_get_str_info(self.handle, "feature_name")
        return v or None

    @feature_names.setter
    def feature_names(self, names):
        if names is not None:
            names = [str(n) for n in names]
            if len(names) != len(set(names)):
                raise ValueError("feature_names must be unique")
            if names and len(names) != self.num_col():
                raise ValueError("feature_names must have the same length as data")
        get_backend().dmatrix_set_str_info(self.handle, "feature_name", names or [])

    @property
    def feature_types(self):
        v = get_backend().dmatrix_get_str_info(self.handle, "feature_type")
        return v or None

    @feature_types.setter
    def feature_types(self, types):
        get_backend().dmatrix_set_str_info(self.handle, "feature_type", list(types) if types else [])


class DataIter:
    """Batches of a QuantileDMatrix (upstream xgboost.DataIter).  Subclasses implement reset() and next(input_data): next passes
    one batch to input_data(data=..., label=..., ...) and returns True, or returns False at the end.  The QuantileDMatrix reads
    the batches twice (once when there is only one), calling reset() before each pass.  A batch is released when next() is
    called again.  cache_prefix, release_data and on_host are accepted for compatibility; the batches are never cached."""

    def __init__(self, cache_prefix=None, release_data=True, *, on_host=True, min_cache_page_bytes=None):
        self.cache_prefix = cache_prefix
        self.release_data = release_data
        self.on_host = on_host
        self.min_cache_page_bytes = min_cache_page_bytes

    def reset(self):
        raise NotImplementedError()

    def next(self, input_data):
        raise NotImplementedError()


_BATCH_FIELDS = ("label", "weight", "base_margin", "qid", "label_lower_bound", "label_upper_bound")


def _set_proxy_batch(be, proxy, data, keep):
    """Hands one batch's features to the proxy; `keep` collects the arrays that must outlive the call."""
    if hasattr(data, "__cuda_array_interface__"):
        iface = data.__cuda_array_interface__
        shape = tuple(iface["shape"])
        if len(shape) != 2:
            raise ValueError("Expecting a 2-dimensional device array, got shape %s" % (shape,))
        contiguous = iface.get("strides") is None or list(iface["strides"]) == [4 * shape[1], 4]
        if iface["typestr"] != "<f4" or not contiguous:           # other layouts are staged as a float32 C-contiguous copy
            if hasattr(data, "contiguous") and hasattr(data, "float"):
                data = data.float().contiguous()
            elif hasattr(data, "astype"):
                data = data.astype("float32", order="C")
            else:
                raise ValueError("device batch must be float32 and C-contiguous")
        keep.append(data)
        be.proxy_set_cuda(proxy, data)
    elif _is_scipy_sparse(data):
        csr = data.tocsr()
        arrs = (np.ascontiguousarray(csr.indptr, dtype=np.uint64), np.ascontiguousarray(csr.indices, dtype=np.uint32),
                np.ascontiguousarray(csr.data, dtype=np.float32))
        keep.extend(arrs)
        be.proxy_set_csr(proxy, *arrs, csr.shape[1])
    else:
        if _is_pandas_df(data):
            arr = data.to_numpy(dtype=np.float32, na_value=np.nan)
        else:
            arr = np.asarray(data)
            if arr.dtype == object or arr.dtype.kind not in "fiub":
                arr = arr.astype(np.float32)
        if arr.ndim == 1:
            arr = arr.reshape(-1, 1)
        if arr.ndim != 2:
            raise ValueError("Expecting 2 dimensional numpy.ndarray, got: %s" % (arr.shape,))
        if arr.dtype == np.float16 or arr.dtype.byteorder == ">":
            arr = arr.astype(np.float32)
        arr = np.ascontiguousarray(arr)
        keep.append(arr)
        be.proxy_set_dense(proxy, arr)


class _SingleBatch(DataIter):
    """In-memory data as an iterator of one batch."""

    def __init__(self, **kwargs):
        super().__init__()
        self._kwargs = kwargs
        self._done = False

    def reset(self):
        self._done = False

    def next(self, input_data):
        if self._done:
            return False
        self._done = True
        input_data(**self._kwargs)
        return True


class QuantileDMatrix(DMatrix):
    """A DMatrix that holds only the binned features (upstream xgboost.QuantileDMatrix): the batches of a DataIter, or in-memory
    data, are binned as they arrive and no float copy of the matrix stays on the device.  max_bin is fixed here (default 256);
    training with another max_bin raises.  ref=: bin with the cuts of that matrix (for evaluation sets).  Prediction reads the
    bins (each value at the lower edge of its bin).  As with DMatrix, a scipy CSR input marks missing values by absence and
    `missing` does not apply to its stored values.  SHAP contributions, booster=dart, process_type=update, slice and xgb.cv
    need the raw features and raise on a QuantileDMatrix."""

    def __init__(self, data, label=None, *, weight=None, base_margin=None, missing=None, silent=False, feature_names=None,
                 feature_types=None, nthread=None, max_bin=None, ref=None, group=None, qid=None, label_lower_bound=None,
                 label_upper_bound=None, feature_weights=None, enable_categorical=False, max_quantile_batches=None,
                 data_split_mode=None):
        self.handle = None
        if enable_categorical:
            raise XGBoostError("categorical features are not supported on the CUDA hist path")
        if feature_weights is not None:
            raise XGBoostError("QuantileDMatrix: feature_weights are not supported on the CUDA hist path")
        if max_bin is None:
            max_bin = 256
        else:
            max_bin = _check_unapplied("max_bin", max_bin)
        if ref is not None and not isinstance(ref, DMatrix):
            raise TypeError("ref must be a DMatrix or a QuantileDMatrix")
        be = get_backend()
        if isinstance(data, DataIter):
            given = dict(label=label, weight=weight, base_margin=base_margin, group=group, qid=qid, label_lower_bound=label_lower_bound,
                         label_upper_bound=label_upper_bound)
            named = [k for k, v in given.items() if v is not None]
            if named:
                raise XGBoostError("QuantileDMatrix(DataIter): pass %s per batch through input_data" % ", ".join(named))
            it = data
        else:
            if group is not None:
                if qid is not None:
                    raise XGBoostError("QuantileDMatrix: give either group or qid")
                sizes = np.asarray(group, dtype=np.int64).reshape(-1)
                qid = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes)
            if feature_names is None and _is_pandas_df(data):
                feature_names = [str(c) for c in data.columns]
            it = _SingleBatch(data=data, label=label, weight=weight, base_margin=base_margin, qid=qid, label_lower_bound=label_lower_bound,
                              label_upper_bound=label_upper_bound)
        if qid is not None:
            _check_ranking_backend()
        proxy = be.proxy_create()
        state = {"keep": [], "error": None, "names": None, "types": None}

        def input_data(data, *, label=None, weight=None, base_margin=None, qid=None, label_lower_bound=None, label_upper_bound=None,
                       feature_names=None, feature_types=None, group=None, **kwargs):
            unknown = [k for k, v in kwargs.items() if v is not None]
            if group is not None or unknown:
                raise XGBoostError("QuantileDMatrix: input_data does not take %s (query groups go per batch as qid)" %
                                   ", ".join((["group"] if group is not None else []) + unknown))
            _set_proxy_batch(be, proxy, data, state["keep"])
            meta = dict(label=label, weight=weight, base_margin=base_margin, qid=qid, label_lower_bound=label_lower_bound,
                        label_upper_bound=label_upper_bound)
            for field in _BATCH_FIELDS:
                v = meta[field]
                if v is None:
                    continue
                if hasattr(v, "__cuda_array_interface__") and hasattr(v, "cpu"):
                    v = v.cpu()
                a = np.asarray(v)
                if field == "qid":
                    a = a if a.dtype.kind in "iu" else a.astype(np.float64)
                else:
                    a = a.astype(np.float32)
                # an (n, T) label with T > 1 keeps its shape: a multi-target label, T the same in every batch
                a = np.ascontiguousarray(a) if field == "label" and a.ndim == 2 and a.shape[1] > 1 else np.ascontiguousarray(a).reshape(-1)
                state["keep"].append(a)
                be.dmatrix_set_info_interface(proxy, field, a)
            if state["names"] is None:
                state["names"] = feature_names if feature_names is not None else ([str(c) for c in data.columns] if _is_pandas_df(data) else None)
                state["types"] = feature_types

        def reset():
            state["keep"] = []
            if state["error"] is None:
                try:
                    it.reset()
                except BaseException as e:  # re-raised once the engine returns
                    state["error"] = e

        def next_():
            state["keep"] = []            # the engine is done with the previous batch
            if state["error"] is not None:
                return False
            try:
                return bool(it.next(input_data))
            except BaseException as e:  # re-raised once the engine returns
                state["error"] = e
                return False

        try:
            h = be.quantile_dmatrix_from_callback(proxy, None if ref is None else ref.handle, reset, next_, missing, max_bin)
        except XGBoostError:
            if state["error"] is not None:        # the iterator's own exception explains the engine's
                raise state["error"]
            raise
        finally:
            state["keep"] = []
            be.dmatrix_free(proxy)
        if state["error"] is not None:
            be.dmatrix_free(h)
            raise state["error"]
        self.handle = h
        self.max_bin = max_bin if ref is None else getattr(ref, "max_bin", max_bin)
        names = feature_names if feature_names is not None else state["names"]
        types = feature_types if feature_types is not None else state["types"]
        if names is not None:
            self.feature_names = names
        if types is not None:
            self.feature_types = types


def _check_ranking_backend():
    if not getattr(get_backend(), "supports_ranking", False):
        raise XGBoostError("query groups (group / qid) and the rank:* objectives are not implemented by this engine")


def _param_items(params):
    """Flatten a params dict / list of pairs the way xgboost.Booster.set_param does (eval_metric lists expand)."""
    if params is None:
        return []
    if isinstance(params, dict):
        items = list(params.items())
    elif isinstance(params, str):
        raise TypeError("params must be a dict or a list of pairs")
    else:
        items = list(params)
    out = []
    for k, v in items:
        if isinstance(v, np.ndarray):          # e.g. quantile_alpha=np.array([0.1, 0.5, 0.9]): forwarded as the list would be
            v = v.tolist() if v.ndim else v.item()
        if k == "eval_metric" and isinstance(v, (list, tuple)):
            out.extend(("eval_metric", m) for m in v)
        elif isinstance(v, (list, tuple)):
            out.append((k, json.dumps(v) if any(isinstance(x, (list, tuple)) for x in v) else "(" + ",".join(str(x) for x in v) + ")"))
        elif isinstance(v, bool):
            out.append((k, "1" if v else "0"))
        elif v is not None:
            out.append((k, v))
    return out


# Parameters the container forwards although they do not concern the hist tree builder; accepted and ignored
# (train.py passes the validated hyperparameter dict through, SURVEY.md section 8b "boundary quirks").
_IGNORED_PARAMS = {
    "csv_weights", "verbosity", "verbose", "silent", "nthread", "n_jobs", "predictor", "sketch_eps", "dsplit", "prob_buffer_row",
    "deterministic_histogram", "single_precision_histogram", "device", "gpu_id",
    "validate_parameters", "max_cat_to_onehot", "max_cat_threshold",
    "lambda_bias", "feature_selector", "top_k",
    "disable_default_eval_metric",
    "max_cached_hist_node", "random_state",
}


_DROP = object()


def _as_float(v, default):
    try:
        return float(v)
    except (TypeError, ValueError):
        return default


def _check_unapplied(k, v):
    """No silent hyperparameter divergence (VERDICT r1): every value the container validates as legal but this builder
    does not honour is either rejected or announced with a warning; returns the value to forward, or _DROP."""
    if k == "monotone_constraints":           # applied (tree.cu constrained_split_gain); forwarded as "(1,0,-1)"
        if isinstance(v, dict):
            raise XGBoostError("monotone_constraints as a feature-name dict is not supported by the CUDA hist builder; pass one entry per feature")
        if isinstance(v, (list, tuple)):
            return "(" + ",".join(str(int(x)) for x in v) + ")"
        return str(v)
    if k == "interaction_constraints":        # applied (tree.cu interaction_children); forwarded as "[[0,1],[2,3,4]]"
        if isinstance(v, (list, tuple)):
            if any(isinstance(x, str) for grp in v for x in (grp if isinstance(grp, (list, tuple)) else [grp])):
                raise XGBoostError("interaction_constraints with feature names are not supported by the CUDA hist builder; use feature indices")
            return "[" + ",".join("[" + ",".join(str(int(x)) for x in grp) + "]" for grp in v) + "]"
        return str(v)
    if k == "max_bin" and _as_float(v, 256) > 256:
        warnings.warn("max_bin=%s exceeds the 256 bins per feature of the uint8 bin codes; using max_bin=256" % v)
        return 256
    if k == "tree_method" and str(v) in ("exact", "approx"):
        warnings.warn("tree_method=%s runs the CUDA hist builder (quantile-binned histograms), not xgboost's %s updater" % (v, v))
        return v
    # process_type=update refreshes / prunes the trees of a loaded model (the engine parses process_type, updater and refresh_leaf,
    # which it ignores under process_type=default); an engine without it must say so rather than grow new trees, and is not sent
    # the three parameters at all
    if k in ("process_type", "updater", "refresh_leaf") and not getattr(get_backend(), "supports_process_type_update", False):
        if k == "process_type" and str(v) == "update":
            raise XGBoostError("process_type=update is not implemented by this engine")
        return _DROP
    if k == "objective" and str(v).startswith("rank:"):
        _check_ranking_backend()
    if k in _IGNORED_PARAMS:
        return _DROP
    return v


class Booster:
    """A gradient-boosted tree model trained / evaluated by the CUDA engine."""

    def __init__(self, params=None, cache=None, model_file=None):
        self.handle = None
        be = get_backend()
        cache = list(cache) if cache else []
        for d in cache:
            if not isinstance(d, DMatrix):
                raise TypeError("invalid cache item: %s" % type(d).__name__)
        self.handle = be.booster_create([d.handle for d in cache])
        self._cache_refs = cache
        if isinstance(model_file, Booster):
            be.booster_unserialize(self.handle, be.booster_serialize(model_file.handle))
        elif isinstance(model_file, (str, os.PathLike)):
            self.load_model(model_file)
        elif isinstance(model_file, (bytes, bytearray)):
            self.load_model(bytearray(model_file))
        elif model_file is not None:
            raise TypeError("Unknown type: %s" % type(model_file).__name__)
        self.set_param(params)

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None:
            try:
                get_backend().booster_free(h)
            except Exception:  # pragma: no cover
                pass
            self.handle = None

    # ---- pickling (serve_utils.py:180-182 tries pickle.load first)
    def __getstate__(self):
        state = {k: v for k, v in self.__dict__.items() if k not in ("handle", "_cache_refs")}
        state["_raw"] = bytearray(get_backend().booster_serialize(self.handle)) if self.handle is not None else None
        return state

    def __setstate__(self, state):
        # Also opens pickles written by xgboost itself (serve_utils.get_loaded_booster tries pickle.load first,
        # algorithm_mode/serve_utils.py:179-181): upstream's state keeps the serialized booster under "handle" (UBJSON
        # {Model, Config} today, "CONFIG-offset:" + the binary model for 1.x) next to plain attributes.
        state = dict(state)
        raw = state.pop("_raw", None)
        if raw is None and isinstance(state.get("handle"), (bytes, bytearray)):
            raw = state["handle"]
        state.pop("handle", None)
        names, types = state.pop("feature_names", None), state.pop("feature_types", None)
        best_it, best_score = state.pop("best_iteration", None), state.pop("best_score", None)
        state.pop("booster", None)                       # 1.x: the booster type ("gbtree"); the document carries it
        self.__dict__.update(state)                      # (1.x also keeps best_ntree_limit, which stays a plain attribute)
        self._cache_refs = []
        self.handle = get_backend().booster_create([])
        if raw is not None:
            get_backend().booster_unserialize(self.handle, bytes(raw))
        if names and self.feature_names is None:
            self.feature_names = names
        if types and self.feature_types is None:
            self.feature_types = types
        if best_it is not None and self.attr("best_iteration") is None:
            self.set_attr(best_iteration=str(best_it))
        if best_score is not None and self.attr("best_score") is None:
            self.set_attr(best_score=str(best_score))

    def __copy__(self):
        return self.copy()

    def __deepcopy__(self, memo):
        return self.copy()

    def copy(self):
        return Booster(model_file=self)

    def __getitem__(self, val):
        if isinstance(val, int):
            val = slice(val, val + 1)
        if not isinstance(val, slice):
            raise TypeError("Booster slicing takes an int or a slice")
        start = val.start or 0
        stop = val.stop or 0
        step = val.step or 1
        if start < 0 or stop < 0 or step < 1:
            raise ValueError("negative indices / steps are not supported")
        total = self.num_boosted_rounds()
        if stop == 0:
            stop = total
        if stop > total or start >= stop:
            raise IndexError("Layer index out of range")
        out = Booster.__new__(Booster)
        out._cache_refs = []
        out.handle = get_backend().booster_slice(self.handle, start, stop, step)
        return out

    # ---- parameters
    def set_param(self, params, value=None):
        if isinstance(params, str) and value is not None:
            params = [(params, value)]
        for k, v in _param_items(params):
            v = _check_unapplied(k, v)
            if v is _DROP:
                continue
            get_backend().booster_set_param(self.handle, k, v)

    def save_config(self):
        return get_backend().booster_save_config(self.handle)

    def load_config(self, config):
        get_backend().booster_load_config(self.handle, config)

    # ---- attributes
    def attr(self, key):
        return get_backend().booster_get_attr(self.handle, key)

    def attributes(self):
        be = get_backend()
        return {k: be.booster_get_attr(self.handle, k) for k in be.booster_attr_names(self.handle)}

    def set_attr(self, **kwargs):
        for k, v in kwargs.items():
            get_backend().booster_set_attr(self.handle, k, None if v is None else str(v))

    @property
    def best_iteration(self):
        v = self.attr("best_iteration")
        if v is None:
            raise AttributeError("`best_iteration` is only defined when early stopping is used.")
        return int(v)

    @best_iteration.setter
    def best_iteration(self, it):
        self.set_attr(best_iteration=it)

    @property
    def best_score(self):
        v = self.attr("best_score")
        if v is None:
            raise AttributeError("`best_score` is only defined when early stopping is used.")
        return float(v)

    @best_score.setter
    def best_score(self, s):
        self.set_attr(best_score=s)

    @property
    def feature_names(self):
        return get_backend().booster_get_str_info(self.handle, "feature_name") or None

    @feature_names.setter
    def feature_names(self, names):
        get_backend().booster_set_str_info(self.handle, "feature_name", [str(n) for n in names] if names else [])

    @property
    def feature_types(self):
        return get_backend().booster_get_str_info(self.handle, "feature_type") or None

    @feature_types.setter
    def feature_types(self, types):
        get_backend().booster_set_str_info(self.handle, "feature_type", list(types) if types else [])

    def num_boosted_rounds(self):
        return get_backend().booster_boosted_rounds(self.handle)

    def num_features(self):
        return get_backend().booster_num_features(self.handle)

    # ---- training
    def _assign_dmatrix_features(self, data):
        if data.num_row() == 0:
            return
        fn, ft = data.feature_names, data.feature_types
        if self.feature_names is None and fn is not None:
            self.feature_names = fn
        if self.feature_types is None and ft is not None:
            self.feature_types = ft

    def _validate_features(self, data):
        if data.num_row() == 0:
            return
        fn = data.feature_names
        mine = self.feature_names
        if mine is None or fn is None:
            if mine is not None and fn is None and len(mine) != data.num_col():
                raise ValueError("feature_names mismatch: training data did not have the following fields: " + ", ".join(mine))
            return
        if list(mine) != list(fn):
            dat_missing = set(mine) - set(fn)
            my_missing = set(fn) - set(mine)
            msg = "feature_names mismatch: {} {}".format(mine, fn)
            if dat_missing:
                msg += "\nexpected " + ", ".join(str(s) for s in dat_missing) + " in input data"
            if my_missing:
                msg += "\ntraining data did not have the following fields: " + ", ".join(str(s) for s in my_missing)
            raise ValueError(msg)

    def update(self, dtrain, iteration, fobj=None):
        if not isinstance(dtrain, DMatrix):
            raise TypeError("invalid training matrix: %s" % type(dtrain).__name__)
        self._assign_dmatrix_features(dtrain)
        if fobj is not None:
            raise XGBoostError("custom objectives are not supported on the CUDA hist path")
        get_backend().booster_update(self.handle, int(iteration), dtrain.handle)

    def boost(self, dtrain, iteration=0, grad=None, hess=None):
        raise XGBoostError("custom objectives (Booster.boost) are not supported on the CUDA hist path")

    def eval_set(self, evals, iteration=0, feval=None, output_margin=True):
        for d, name in evals:
            if not isinstance(d, DMatrix):
                raise TypeError("expected DMatrix, got %s" % type(d).__name__)
            if not isinstance(name, str):
                raise TypeError("expected string, got %s" % type(name).__name__)
            self._validate_features(d)
        msg = get_backend().booster_eval(self.handle, int(iteration), [d.handle for d, _ in evals], [n for _, n in evals])
        if feval is not None:
            from . import container_metrics
            names = container_metrics.recognise(feval) if container_metrics.device_route_available() else None
            for dmat, evname in evals:
                if names is not None:         # the container's own metrics: finished from the engine's exact raw results
                    feval_ret = container_metrics.evaluate(self, dmat, names, output_margin)
                else:
                    feval_ret = feval(self.predict(dmat, training=False, output_margin=output_margin), dmat)
                if isinstance(feval_ret, list):
                    for name, val in feval_ret:
                        msg += "\t%s-%s:%f" % (evname, name, val)
                else:
                    name, val = feval_ret
                    msg += "\t%s-%s:%f" % (evname, name, val)
        return msg

    def eval(self, data, name="eval", iteration=0):
        self._validate_features(data)
        return self.eval_set([(data, name)], iteration)

    # ---- inference
    def predict(self, data, output_margin=False, pred_leaf=False, pred_contribs=False, approx_contribs=False,
                pred_interactions=False, validate_features=True, training=False, iteration_range=(0, 0), strict_shape=False):
        if not isinstance(data, DMatrix):
            raise TypeError("Expecting data to be a DMatrix object, got: %s" % type(data))
        if validate_features:
            self._validate_features(data)
        if approx_contribs or pred_interactions:
            raise XGBoostError("approx_contribs / pred_interactions are not implemented on the CUDA path (pred_contribs is)")
        ptype = 1 if output_margin else 0
        if pred_leaf:
            ptype = 6
        if pred_contribs:
            ptype = 2           # exact path-dependent Tree SHAP on the device, shape (n, F + 1) or (n, K, F + 1); last column = bias
        cfg = {"type": ptype, "training": bool(training), "iteration_begin": int(iteration_range[0]),
               "iteration_end": int(iteration_range[1]), "strict_shape": bool(strict_shape)}
        return get_backend().booster_predict(self.handle, data.handle, cfg)

    # ---- model IO
    def save_raw(self, raw_format="ubj"):
        if raw_format == "deprecated":
            raise XGBoostError("writing the legacy binary model format is not supported (it is read by load_model); use 'ubj' or 'json'")
        return bytearray(get_backend().booster_save_raw(self.handle, raw_format))

    def save_model(self, fname):
        if not isinstance(fname, (str, os.PathLike)):
            raise TypeError("fname must be a string or os PathLike")
        fname = os.fspath(os.path.expanduser(fname))
        fmt = "json" if fname.endswith(".json") else "ubj"
        raw = get_backend().booster_save_raw(self.handle, fmt)
        try:
            with open(fname, "wb") as f:
                f.write(raw)
        except OSError as e:
            raise XGBoostError("Opening %s failed: %s" % (fname, e))

    def load_model(self, fname):
        if isinstance(fname, (str, os.PathLike)):
            fname = os.fspath(os.path.expanduser(fname))
            try:
                with open(fname, "rb") as f:
                    buf = f.read()
            except OSError as e:
                raise XGBoostError("Opening %s failed: %s" % (fname, e))
        elif isinstance(fname, (bytes, bytearray)):
            buf = bytes(fname)
        else:
            raise TypeError("Unknown file type: %s" % type(fname).__name__)
        get_backend().booster_load_raw(self.handle, buf)

    def get_dump(self, fmap="", with_stats=False, dump_format="text"):
        """Text / JSON dump of the trees (subset of upstream's formats, enough for inspection and tests)."""
        m = get_backend().booster_export_model(self.handle) if hasattr(get_backend(), "booster_export_model") else None
        if m is None:
            raise XGBoostError("get_dump is unavailable with this backend")
        names = self.feature_names
        out = []
        for t in range(len(m["tree_info"])):
            a = int(m["tree_offset"][t])

            def rec(i, depth):
                gi = a + i
                if m["left"][gi] == -1:
                    s = "%s%d:leaf=%.9g" % ("\t" * depth, i, m["split_cond"][gi])
                    if with_stats:
                        s += ",cover=%.9g" % m["sum_hess"][gi]
                    return s + "\n"
                f = int(m["split_index"][gi])
                fname = names[f] if names else "f%d" % f
                l, r = int(m["left"][gi]), int(m["right"][gi])
                miss = l if m["default_left"][gi] else r
                s = "%s%d:[%s<%.9g] yes=%d,no=%d,missing=%d" % ("\t" * depth, i, fname, m["split_cond"][gi], l, r, miss)
                if with_stats:
                    s += ",gain=%.9g,cover=%.9g" % (m["loss_chg"][gi], m["sum_hess"][gi])
                return s + "\n" + rec(l, depth + 1) + rec(r, depth + 1)

            out.append(rec(0, 0))
        return out

    def get_score(self, fmap="", importance_type="weight"):
        m = get_backend().booster_export_model(self.handle)
        names = self.feature_names
        internal = m["left"] != -1
        res = {}
        for gi in np.nonzero(internal)[0]:
            f = int(m["split_index"][gi])
            key = names[f] if names else "f%d" % f
            w, g, c = res.get(key, (0, 0.0, 0.0))
            res[key] = (w + 1, g + float(m["loss_chg"][gi]), c + float(m["sum_hess"][gi]))
        if importance_type == "weight":
            return {k: float(v[0]) for k, v in res.items()}
        if importance_type == "gain":
            return {k: v[1] / v[0] for k, v in res.items()}
        if importance_type == "cover":
            return {k: v[2] / v[0] for k, v in res.items()}
        if importance_type == "total_gain":
            return {k: v[1] for k, v in res.items()}
        if importance_type == "total_cover":
            return {k: v[2] for k, v in res.items()}
        raise ValueError("Unknown importance type: %s" % importance_type)
