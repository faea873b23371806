"""ctypes binding of libb200xgb.so (include/b200xgb.h) -- the only compute backend of this package.

The functions bound here carry the names and conventions of libxgboost's C API, i.e. what the reference
container reaches through `import xgboost` (SURVEY.md section 8b).  There is deliberately NO CPU fallback: if the
CUDA library is missing, or no GPU is visible, every call fails loudly with XGBoostError.
"""
import ctypes as C
import json
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200xgb.so")

c_bst_ulong = C.c_uint64


class XGBoostError(ValueError):
    """Error raised by the native library (same name and base class as xgboost.core.XGBoostError)."""


def _cstr(s):
    return C.c_char_p(s.encode("utf-8"))


def _from_cstr_array(ptr, n):
    return [ptr[i].decode("utf-8") for i in range(n)]


_utf8_and_size = C.pythonapi.PyUnicode_AsUTF8AndSize
_utf8_and_size.restype = C.c_void_p
_utf8_and_size.argtypes = [C.py_object, C.POINTER(C.c_ssize_t)]


class CudaBackend:
    """Thin, stateless wrapper: one method per C-ABI entry point."""

    name = "cuda"
    supports_process_type_update = True      # refresh / prune of loaded trees (csrc/refresh.cu)
    supports_ranking = True                  # query groups, rank:* objectives, ndcg / map metrics (csrc/rank.cu)

    def __init__(self, path=LIB_PATH):
        if not os.path.exists(path):
            raise XGBoostError(
                "libb200xgb.so not found at %s -- build it with `python sagemaker-xgboost-container_b200/build.py` "
                "(nvcc, sm_90a). This package has no CPU fallback." % path)
        self.lib = C.CDLL(path)
        self.lib.XGBGetLastError.restype = C.c_char_p
        self.path = path

    # ------------------------------------------------------------------ helpers
    def _check(self, ret):
        if ret != 0:
            raise XGBoostError(self.lib.XGBGetLastError().decode("utf-8", "replace"))

    def build_info(self):
        out = C.c_char_p()
        self._check(self.lib.XGBuildInfo(C.byref(out)))
        return json.loads(out.value.decode())

    # ------------------------------------------------------------------ DMatrix
    def dmatrix_from_dense(self, arr, missing):
        arr = np.ascontiguousarray(arr, dtype=np.float32)
        if arr.ndim != 2:
            raise ValueError("Expecting 2 dimensional numpy.ndarray, got: %s" % (arr.shape,))
        h = C.c_void_p()
        self._check(self.lib.XGDMatrixCreateFromMat(arr.ctypes.data_as(C.POINTER(C.c_float)), c_bst_ulong(arr.shape[0]),
                                                    c_bst_ulong(arr.shape[1]), C.c_float(missing), C.byref(h)))
        return h

    def dmatrix_from_csr(self, indptr, indices, data, ncol):
        indptr = np.ascontiguousarray(indptr, dtype=np.uint64)
        indices = np.ascontiguousarray(indices, dtype=np.uint32)
        data = np.ascontiguousarray(data, dtype=np.float32)
        h = C.c_void_p()
        self._check(self.lib.XGDMatrixCreateFromCSREx(indptr.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                      indices.ctypes.data_as(C.POINTER(C.c_uint)),
                                                      data.ctypes.data_as(C.POINTER(C.c_float)), C.c_size_t(len(indptr)),
                                                      C.c_size_t(len(data)), C.c_size_t(ncol), C.byref(h)))
        return h

    def dmatrix_from_cuda_array(self, obj, missing):
        """obj exposes __cuda_array_interface__ (torch.Tensor on cuda, cupy.ndarray): float32, 2-D, C-contiguous."""
        iface = dict(obj.__cuda_array_interface__)
        iface["shape"] = list(iface["shape"])
        iface["data"] = [int(iface["data"][0]), bool(iface["data"][1])]
        iface.pop("stream", None)
        iface["strides"] = None if iface.get("strides") is None else list(iface["strides"])
        if iface["strides"] is not None:
            n, F = iface["shape"]
            if list(iface["strides"]) != [4 * F, 4]:
                raise ValueError("device array must be C-contiguous")
            iface["strides"] = None
        h = C.c_void_p()
        cfg = {} if missing is None or missing != missing else {"missing": float(missing)}
        self._check(self.lib.XGDMatrixCreateFromCudaArrayInterface(_cstr(json.dumps(iface)), _cstr(json.dumps(cfg)), C.byref(h)))
        return h

    # ------------------------------------------------------------------ QuantileDMatrix (proxy batches + callbacks)
    _RESET_CB = C.CFUNCTYPE(None, C.c_void_p)
    _NEXT_CB = C.CFUNCTYPE(C.c_int, C.c_void_p)

    def proxy_create(self):
        h = C.c_void_p()
        self._check(self.lib.XGProxyDMatrixCreate(C.byref(h)))
        return h

    @staticmethod
    def _host_iface(arr):
        return json.dumps({"data": [int(arr.ctypes.data), True], "shape": list(arr.shape), "typestr": arr.dtype.str, "version": 3})

    def proxy_set_dense(self, h, arr):
        """arr: 2-D C-contiguous numpy array of a numeric dtype (kept alive by the caller until the next batch)."""
        self._check(self.lib.XGProxyDMatrixSetDataDense(h, _cstr(self._host_iface(arr))))

    def proxy_set_cuda(self, h, obj):
        """obj exposes __cuda_array_interface__: float32, 2-D, C-contiguous (read in place)."""
        iface = dict(obj.__cuda_array_interface__)
        n, F = iface["shape"]
        if iface["typestr"] != "<f4" or (iface.get("strides") is not None and list(iface["strides"]) != [4 * F, 4]):
            raise ValueError("device batch must be float32 and C-contiguous")
        out = {"data": [int(iface["data"][0]), bool(iface["data"][1])], "shape": [int(n), int(F)], "typestr": "<f4", "strides": None, "version": 3}
        self._check(self.lib.XGProxyDMatrixSetDataCudaArrayInterface(h, _cstr(json.dumps(out))))

    def proxy_set_csr(self, h, indptr, indices, data, ncol):
        self._check(self.lib.XGProxyDMatrixSetDataCSR(h, _cstr(self._host_iface(indptr)), _cstr(self._host_iface(indices)),
                                                      _cstr(self._host_iface(data)), c_bst_ulong(ncol)))

    def quantile_dmatrix_from_callback(self, proxy, ref, reset, next_, missing, max_bin):
        """reset() / next_() -> bool are Python callables; next_ sets the batch on `proxy` before it returns True."""
        reset_cb = self._RESET_CB(lambda _: reset())
        next_cb = self._NEXT_CB(lambda _: 1 if next_() else 0)
        cfg = {"max_bin": int(max_bin)}
        if missing is not None and missing == missing:
            cfg["missing"] = float(missing)
        h = C.c_void_p()
        self._check(self.lib.XGQuantileDMatrixCreateFromCallback(None, proxy, ref, reset_cb, next_cb, _cstr(json.dumps(cfg)), C.byref(h)))
        return h

    def device_memory(self, reset_peak=False):
        """(live, peak) bytes the engine holds in its device buffers (XGB200DeviceMemory)."""
        live, peak = c_bst_ulong(), c_bst_ulong()
        self._check(self.lib.XGB200DeviceMemory(C.byref(live), C.byref(peak), C.c_int(1 if reset_peak else 0)))
        return int(live.value), int(peak.value)

    def dmatrix_get_raw(self, h):
        n, F = self.dmatrix_num_row(h), self.dmatrix_num_col(h)
        out = np.empty(n * F, np.float32)
        self._check(self.lib.XGB200DMatrixGetRaw(h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def dmatrix_from_csv_labeled(self, payload, delimiter=",", label_column=-1, weight_column=-1):
        """Device-side parse of a training CSV channel; (handle, status) like dmatrix_from_csv."""
        h = C.c_void_p()
        st = C.c_int(0)
        self._check(self.lib.XGB200DMatrixCreateFromCSVEx(C.c_char_p(payload), C.c_ulong(len(payload)), C.c_char(delimiter.encode("ascii")),
                                                          C.c_int(label_column), C.c_int(weight_column), C.byref(st), C.byref(h)))
        return (h if st.value == 0 else None), int(st.value)

    _COL_TYPES = {"<f4": 0, "<f8": 1, "<i4": 2, "<i8": 3, "|u1": 4, "|i1": 5, "<i2": 6, "<u2": 7, "<u4": 8, "<u8": 9, "|b1": 10}

    def dmatrix_from_columns(self, columns, label_column=-1, weight_column=-1):
        """Columnar input (ingest.cu): one contiguous 1-D numpy array per column, in its own dtype where the device converts it
        (float32/64, (u)int8..64, bool), anything else converted to float32 one column at a time -- never a dense host matrix."""
        cols = []
        for c in columns:
            a = np.asarray(c)
            if a.ndim != 1:
                raise ValueError("columns must be 1-dimensional")
            if a.dtype.str not in self._COL_TYPES:
                a = a.astype(np.float32)
            cols.append(np.ascontiguousarray(a))
        n = len(cols[0]) if cols else 0
        if any(len(a) != n for a in cols):
            raise ValueError("columns have different lengths")
        ptrs = (C.c_void_p * len(cols))(*[a.ctypes.data for a in cols])
        types = (C.c_int * len(cols))(*[self._COL_TYPES[a.dtype.str] for a in cols])
        h = C.c_void_p()
        self._check(self.lib.XGB200DMatrixCreateFromColumns(ptrs, types, C.c_int(len(cols)), C.c_ulong(n), C.c_int(label_column), C.c_int(weight_column), C.byref(h)))
        return h

    def dmatrix_from_libsvm_text(self, payload, whitespace_mode, absent):
        """Device-side parse of a libsvm request body (csv.cu).  Returns (handle, status); handle is None unless status == 0."""
        h = C.c_void_p()
        st = C.c_int(0)
        if isinstance(payload, str):
            size = C.c_ssize_t(0)
            ptr = _utf8_and_size(payload, C.byref(size))
            if not ptr:
                raise ValueError("libsvm payload is not valid UTF-8")
            text, length = C.c_char_p(ptr), size.value
        else:
            text, length = C.c_char_p(bytes(payload) if not isinstance(payload, bytes) else payload), len(payload)
        self._check(self.lib.XGB200DMatrixCreateFromLibsvmText(text, C.c_ulong(length), C.c_int(whitespace_mode), C.c_float(absent), C.byref(st), C.byref(h)))
        return (h if st.value == 0 else None), int(st.value)

    def dmatrix_from_recordio(self, buf):
        """Device-side decode of a recordio-protobuf body (recordio.cu).  Returns (handle, status, message); handle is None
        unless status == 0, message names the rule the body breaks when status == 1 (include/b200xgb.h)."""
        body = np.frombuffer(buf, np.uint8)              # bytes / bytearray / memoryview without a copy
        h = C.c_void_p()
        st = C.c_int(0)
        self._check(self.lib.XGB200DMatrixCreateFromRecordIO(C.c_void_p(body.ctypes.data if body.size else None), c_bst_ulong(body.size),
                                                             C.byref(st), C.byref(h)))
        message = self.lib.XGBGetLastError().decode("utf-8", "replace") if st.value == 1 else ""
        return (h if st.value == 0 else None), int(st.value), message

    def dmatrix_from_csv(self, payload, delimiter=","):
        """Device-side CSV parse (csv.cu).  Returns (handle, status); handle is None unless status == 0."""
        h = C.c_void_p()
        st = C.c_int(0)
        if isinstance(payload, str):
            # CPython caches the UTF-8 form of a str (for ASCII text it IS the object's own buffer): no 200 MB .encode() copy
            size = C.c_ssize_t(0)
            ptr = _utf8_and_size(payload, C.byref(size))
            if not ptr:
                raise ValueError("CSV payload is not valid UTF-8")
            text, length = C.c_char_p(ptr), size.value
        else:
            text, length = C.c_char_p(bytes(payload) if not isinstance(payload, bytes) else payload), len(payload)
        self._check(self.lib.XGB200DMatrixCreateFromCSV(text, C.c_ulong(length), C.c_char(delimiter.encode("ascii")), C.byref(st), C.byref(h)))
        return (h if st.value == 0 else None), int(st.value)

    def dmatrix_free(self, h):
        self._check(self.lib.XGDMatrixFree(h))

    def dmatrix_num_row(self, h):
        out = c_bst_ulong()
        self._check(self.lib.XGDMatrixNumRow(h, C.byref(out)))
        return int(out.value)

    def dmatrix_num_col(self, h):
        out = c_bst_ulong()
        self._check(self.lib.XGDMatrixNumCol(h, C.byref(out)))
        return int(out.value)

    def dmatrix_set_float_info(self, h, field, arr):
        arr = np.ascontiguousarray(arr, dtype=np.float32).reshape(-1)
        self._check(self.lib.XGDMatrixSetFloatInfo(h, _cstr(field), arr.ctypes.data_as(C.POINTER(C.c_float)), c_bst_ulong(arr.size)))

    def dmatrix_get_float_info(self, h, field):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_float)()
        self._check(self.lib.XGDMatrixGetFloatInfo(h, _cstr(field), C.byref(n), C.byref(ptr)))
        if n.value == 0:
            return np.zeros(0, np.float32)
        return np.ctypeslib.as_array(ptr, shape=(n.value,)).copy()

    def dmatrix_slice(self, h, idx, allow_groups=False):
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        out = C.c_void_p()
        self._check(self.lib.XGDMatrixSliceDMatrixEx(h, idx.ctypes.data_as(C.POINTER(C.c_int)), c_bst_ulong(len(idx)), C.byref(out),
                                                     C.c_int(1 if allow_groups else 0)))
        return out

    def dmatrix_set_info_interface(self, h, field, arr):
        """XGDMatrixSetInfoFromInterface with a host array (upstream's route for "group" and "qid"): 1-D, or a 2-D (n, T) label."""
        arr = np.ascontiguousarray(arr)
        if arr.ndim != 2:
            arr = arr.reshape(-1)
        iface = {"data": [int(arr.ctypes.data), True], "shape": [int(d) for d in arr.shape], "typestr": arr.dtype.str, "version": 3}
        self._check(self.lib.XGDMatrixSetInfoFromInterface(h, _cstr(field), _cstr(json.dumps(iface))))

    def dmatrix_set_uint_info(self, h, field, arr):
        arr = np.ascontiguousarray(arr, dtype=np.uint32).reshape(-1)
        self._check(self.lib.XGDMatrixSetUIntInfo(h, _cstr(field), arr.ctypes.data_as(C.POINTER(C.c_uint)), c_bst_ulong(arr.size)))

    def dmatrix_set_group(self, h, sizes):
        arr = np.ascontiguousarray(sizes, dtype=np.uint32).reshape(-1)
        self._check(self.lib.XGDMatrixSetGroup(h, arr.ctypes.data_as(C.POINTER(C.c_uint)), c_bst_ulong(arr.size)))

    def dmatrix_get_uint_info(self, h, field):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_uint)()
        self._check(self.lib.XGDMatrixGetUIntInfo(h, _cstr(field), C.byref(n), C.byref(ptr)))
        if n.value == 0:
            return np.zeros(0, np.uint32)
        return np.ctypeslib.as_array(ptr, shape=(n.value,)).copy()

    def dmatrix_set_str_info(self, h, field, values):
        values = list(values or [])
        arr = (C.c_char_p * len(values))(*[v.encode("utf-8") for v in values])
        self._check(self.lib.XGDMatrixSetStrFeatureInfo(h, _cstr(field), arr, c_bst_ulong(len(values))))

    def dmatrix_get_str_info(self, h, field):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_char_p)()
        self._check(self.lib.XGDMatrixGetStrFeatureInfo(h, _cstr(field), C.byref(n), C.byref(ptr)))
        return _from_cstr_array(ptr, n.value)

    # ------------------------------------------------------------------ Booster
    def booster_create(self, dmat_handles=()):
        arr = (C.c_void_p * len(dmat_handles))(*[d.value if isinstance(d, C.c_void_p) else d for d in dmat_handles])
        h = C.c_void_p()
        self._check(self.lib.XGBoosterCreate(arr, c_bst_ulong(len(dmat_handles)), C.byref(h)))
        return h

    def booster_free(self, h):
        self._check(self.lib.XGBoosterFree(h))

    def booster_set_param(self, h, k, v):
        self._check(self.lib.XGBoosterSetParam(h, _cstr(str(k)), _cstr(str(v))))

    def booster_update(self, h, it, dh):
        self._check(self.lib.XGBoosterUpdateOneIter(h, C.c_int(it), dh))

    def booster_eval(self, h, it, dhs, names):
        dm = (C.c_void_p * len(dhs))(*[d.value for d in dhs])
        nm = (C.c_char_p * len(names))(*[n.encode("utf-8") for n in names])
        out = C.c_char_p()
        self._check(self.lib.XGBoosterEvalOneIter(h, C.c_int(it), dm, nm, c_bst_ulong(len(dhs)), C.byref(out)))
        return out.value.decode("utf-8")

    def booster_predict(self, h, dh, cfg):
        shape = C.POINTER(c_bst_ulong)()
        dim = c_bst_ulong()
        res = C.POINTER(C.c_float)()
        self._check(self.lib.XGBoosterPredictFromDMatrix(h, dh, _cstr(json.dumps(cfg)), C.byref(shape), C.byref(dim), C.byref(res)))
        shp = tuple(int(shape[i]) for i in range(dim.value))
        n = int(np.prod(shp)) if shp else 0
        if n == 0:
            return np.zeros(shp, np.float32)
        return np.ctypeslib.as_array(res, shape=(n,)).copy().reshape(shp)

    def booster_save_raw(self, h, fmt):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_char)()
        self._check(self.lib.XGBoosterSaveModelToBuffer(h, _cstr(json.dumps({"format": fmt})), C.byref(n), C.byref(ptr)))
        return C.string_at(ptr, n.value)

    def booster_load_raw(self, h, buf):
        buf = bytes(buf)
        self._check(self.lib.XGBoosterLoadModelFromBuffer(h, buf, c_bst_ulong(len(buf))))

    def booster_serialize(self, h):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_char)()
        self._check(self.lib.XGBoosterSerializeToBuffer(h, C.byref(n), C.byref(ptr)))
        return C.string_at(ptr, n.value)

    def booster_unserialize(self, h, buf):
        buf = bytes(buf)
        self._check(self.lib.XGBoosterUnserializeFromBuffer(h, buf, c_bst_ulong(len(buf))))

    def booster_save_config(self, h):
        n = c_bst_ulong()
        out = C.c_char_p()
        self._check(self.lib.XGBoosterSaveJsonConfig(h, C.byref(n), C.byref(out)))
        return out.value.decode("utf-8")

    def booster_load_config(self, h, s):
        self._check(self.lib.XGBoosterLoadJsonConfig(h, _cstr(s)))

    def booster_num_features(self, h):
        out = c_bst_ulong()
        self._check(self.lib.XGBoosterGetNumFeature(h, C.byref(out)))
        return int(out.value)

    def booster_boosted_rounds(self, h):
        out = C.c_int()
        self._check(self.lib.XGBoosterBoostedRounds(h, C.byref(out)))
        return int(out.value)

    def booster_slice(self, h, begin, end, step):
        out = C.c_void_p()
        self._check(self.lib.XGBoosterSlice(h, C.c_int(begin), C.c_int(end), C.c_int(step), C.byref(out)))
        return out

    def booster_get_attr(self, h, key):
        out = C.c_char_p()
        ok = C.c_int()
        self._check(self.lib.XGBoosterGetAttr(h, _cstr(key), C.byref(out), C.byref(ok)))
        return out.value.decode("utf-8") if ok.value else None

    def booster_set_attr(self, h, key, value):
        self._check(self.lib.XGBoosterSetAttr(h, _cstr(key), None if value is None else _cstr(str(value))))

    def booster_attr_names(self, h):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_char_p)()
        self._check(self.lib.XGBoosterGetAttrNames(h, C.byref(n), C.byref(ptr)))
        return _from_cstr_array(ptr, n.value)

    def booster_set_str_info(self, h, field, values):
        values = list(values or [])
        arr = (C.c_char_p * len(values))(*[v.encode("utf-8") for v in values])
        self._check(self.lib.XGBoosterSetStrFeatureInfo(h, _cstr(field), arr, c_bst_ulong(len(values))))

    def booster_get_str_info(self, h, field):
        n = c_bst_ulong()
        ptr = C.POINTER(C.c_char_p)()
        self._check(self.lib.XGBoosterGetStrFeatureInfo(h, _cstr(field), C.byref(n), C.byref(ptr)))
        return _from_cstr_array(ptr, n.value)

    # ------------------------------------------------------------------ collective
    def comm_unique_id(self):
        out = C.c_char_p()
        self._check(self.lib.XGCommunicatorGetUniqueId(C.byref(out)))
        return out.value.decode()

    def comm_init(self, cfg):
        self._check(self.lib.XGCommunicatorInit(_cstr(json.dumps(cfg))))

    def comm_finalize(self):
        self._check(self.lib.XGCommunicatorFinalize())

    def comm_peer_reduce_active(self):
        return bool(self.lib.XGB200CommPeerReduceActive())

    def comm_rank(self):
        return int(self.lib.XGCommunicatorGetRank())

    def comm_world(self):
        return int(self.lib.XGCommunicatorGetWorldSize())

    # ------------------------------------------------------------------ introspection (tests / bench)
    def dmatrix_get_cuts(self, h, max_bin):
        n_ptrs, n_vals = c_bst_ulong(), c_bst_ulong()
        ptrs, vals, mins = C.POINTER(C.c_int)(), C.POINTER(C.c_float)(), C.POINTER(C.c_float)()
        hm = C.c_int()
        self._check(self.lib.XGB200DMatrixGetCuts(h, C.c_int(max_bin), C.byref(n_ptrs), C.byref(ptrs), C.byref(n_vals), C.byref(vals),
                                                  C.byref(mins), C.byref(hm)))
        F = n_ptrs.value - 1
        return (np.ctypeslib.as_array(ptrs, shape=(n_ptrs.value,)).copy(), np.ctypeslib.as_array(vals, shape=(n_vals.value,)).copy(),
                np.ctypeslib.as_array(mins, shape=(F,)).copy() if F else np.zeros(0, np.float32), bool(hm.value))

    def dmatrix_set_cuts(self, h, ptrs, vals, mins):
        ptrs = np.ascontiguousarray(ptrs, np.int32)
        vals = np.ascontiguousarray(vals, np.float32)
        mins = np.ascontiguousarray(mins, np.float32)
        self._check(self.lib.XGB200DMatrixSetCuts(h, ptrs.ctypes.data_as(C.POINTER(C.c_int)), c_bst_ulong(len(ptrs)),
                                                  vals.ctypes.data_as(C.POINTER(C.c_float)), mins.ctypes.data_as(C.POINTER(C.c_float))))

    def dmatrix_get_bins(self, h, max_bin):
        n, F = self.dmatrix_num_row(h), self.dmatrix_num_col(h)
        out = np.zeros((n, F), np.uint8)
        self._check(self.lib.XGB200DMatrixGetBins(h, C.c_int(max_bin), out.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out

    def dmatrix_get_bin_copies(self, h, max_bin):
        """(aligned, col): the 128 B line-aligned row copy as [n][128] uint8 (None when the matrix has none) and the
        column-major copy as [F][n] uint8 (include/b200xgb.h XGB200DMatrixGetBinCopies)."""
        n, F = self.dmatrix_num_row(h), self.dmatrix_num_col(h)
        stride = C.c_int()
        self._check(self.lib.XGB200DMatrixGetBinCopies(h, C.c_int(max_bin), C.byref(stride), None, None))
        aligned = np.zeros((n, stride.value), np.uint8) if stride.value else None
        col = np.zeros((F, n), np.uint8)
        u8 = C.POINTER(C.c_uint8)
        self._check(self.lib.XGB200DMatrixGetBinCopies(h, C.c_int(max_bin), C.byref(stride),
                                                       aligned.ctypes.data_as(u8) if aligned is not None else None, col.ctypes.data_as(u8)))
        return aligned, col

    def dmatrix_rank_cuts(self, h, max_bin, row_bounds):
        """Cuts of the multi-GPU recipe with rows [row_bounds[r], row_bounds[r+1]) as rank r's shard: (ptrs, vals, mins)
        (include/b200xgb.h XGB200DMatrixRankCuts)."""
        F = self.dmatrix_num_col(h)
        bounds = np.ascontiguousarray(row_bounds, np.int64)
        ptrs = np.zeros(F + 1, np.int32)
        vals = np.zeros(max(F, 1) * 256, np.float32)
        mins = np.zeros(max(F, 1), np.float32)
        self._check(self.lib.XGB200DMatrixRankCuts(h, C.c_int(max_bin), bounds.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(bounds) - 1),
                                                   ptrs.ctypes.data_as(C.POINTER(C.c_int)), vals.ctypes.data_as(C.POINTER(C.c_float)),
                                                   mins.ctypes.data_as(C.POINTER(C.c_float))))
        return ptrs, vals[:ptrs[-1]].copy(), mins[:F].copy()

    def segmented_quantile(self, values, segments=None, weights=None, n_segments=1, alpha=0.5):
        """The alpha-quantile of each segment with the select kernels of reg:absoluteerror's leaf refresh: float32 (n_segments,),
        NaN for an empty segment (include/b200xgb.h XGB200SegmentedQuantile)."""
        v = np.ascontiguousarray(values, np.float32)
        seg = None if segments is None else np.ascontiguousarray(segments, np.int32)
        w = None if weights is None else np.ascontiguousarray(weights, np.float32)
        out = np.zeros(int(n_segments), np.float32)
        fp = C.POINTER(C.c_float)
        self._check(self.lib.XGB200SegmentedQuantile(v.ctypes.data_as(fp), None if seg is None else seg.ctypes.data_as(C.POINTER(C.c_int32)),
                                                     None if w is None else w.ctypes.data_as(fp), c_bst_ulong(len(v)), C.c_int(int(n_segments)),
                                                     C.c_float(alpha), out.ctypes.data_as(fp)))
        return out

    def gradient_based_sample(self, gpair, subsample, seed=0, stream=0x2000):
        """sampling_method=gradient_based on the given (n, 2) pairs with the training kernels: (threshold u, sampled pairs (n, 2))
        (include/b200xgb.h XGB200GradientBasedSample)."""
        gp = np.ascontiguousarray(gpair, np.float32).reshape(-1, 2)
        out = np.zeros_like(gp)
        u = C.c_float()
        fp = C.POINTER(C.c_float)
        self._check(self.lib.XGB200GradientBasedSample(gp.ctypes.data_as(fp), c_bst_ulong(len(gp)), C.c_float(subsample), C.c_uint(int(seed)),
                                                       C.c_uint64(int(stream)), C.byref(u), out.ctypes.data_as(fp)))
        return np.float32(u.value), out

    def booster_export_model(self, h):
        nt, nn = c_bst_ulong(), c_bst_ulong()
        bs = C.c_float()
        nc = C.c_int()
        self._check(self.lib.XGB200BoosterModelShape(h, C.byref(nt), C.byref(nn), C.byref(bs), C.byref(nc)))
        nt, nn = nt.value, nn.value
        m = {"tree_offset": np.zeros(nt + 1, np.int64), "tree_info": np.zeros(nt, np.int32)}
        for k in ("left", "right", "parent", "split_index", "split_bin"):
            m[k] = np.zeros(nn, np.int32)
        m["default_left"] = np.zeros(nn, np.uint8)
        for k in ("split_cond", "base_weight", "loss_chg", "sum_hess"):
            m[k] = np.zeros(nn, np.float32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self._check(self.lib.XGB200BoosterExportModel(h, p(m["tree_offset"]), p(m["tree_info"]), p(m["left"]), p(m["right"]), p(m["parent"]),
                                                      p(m["split_index"]), p(m["split_bin"]), p(m["default_left"]), p(m["split_cond"]),
                                                      p(m["base_weight"]), p(m["loss_chg"]), p(m["sum_hess"])))
        m["base_score"] = float(bs.value)
        m["num_class"] = int(nc.value)
        return m

    def build_root_histogram(self, bh, dh, gpair, repeats=1):
        gpair = np.ascontiguousarray(gpair, np.float32)
        F = self.dmatrix_num_col(dh)
        hist = np.zeros((F, 256, 2), np.int64)
        scales = np.zeros(4, np.float32)
        ms = C.c_float()
        self._check(self.lib.XGB200BuildRootHistogram(bh, dh, gpair.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(repeats),
                                                      hist.ctypes.data_as(C.POINTER(C.c_int64)), scales.ctypes.data_as(C.POINTER(C.c_float)),
                                                      C.byref(ms)))
        return hist, scales, float(ms.value)

    def build_histogram_ex(self, bh, dh, gpair, mode=0, row_ids=None, repeats=1):
        """Kernel-level entry point: (hist [F][256][2] int64, scales, ms, kernel name); see include/b200xgb.h."""
        gpair = np.ascontiguousarray(gpair, np.float32)
        F = self.dmatrix_num_col(dh)
        hist = np.zeros((F, 256, 2), np.int64)
        scales = np.zeros(4, np.float32)
        ms = C.c_float()
        name = C.c_char_p()
        ids, n_ids = None, 0
        if row_ids is not None:
            row_ids = np.ascontiguousarray(row_ids, np.uint32)
            ids, n_ids = row_ids.ctypes.data_as(C.POINTER(C.c_uint)), len(row_ids)
        self._check(self.lib.XGB200BuildHistogramEx(bh, dh, gpair.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(repeats), C.c_int(mode), ids,
                                                    C.c_ulong(n_ids), hist.ctypes.data_as(C.POINTER(C.c_int64)),
                                                    scales.ctypes.data_as(C.POINTER(C.c_float)), C.byref(ms), C.byref(name)))
        return hist, scales, float(ms.value), (name.value or b"").decode()

    def eval_root_split(self, bh, dh, hist, G, H, max_g, max_h, lower=float("-inf"), upper=float("inf"), feat_mask=None):
        """Split evaluation of one root from an int64 [F][256][2] histogram (include/b200xgb.h XGB200BoosterEvalRootSplit):
        a dict whose floats are uint32 bit patterns."""
        hist = np.ascontiguousarray(hist, np.int64)
        mask = None if feat_mask is None else np.ascontiguousarray(feat_mask, np.uint8)
        out = C.c_char_p()
        self._check(self.lib.XGB200BoosterEvalRootSplit(bh, dh, hist.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(int(G)), C.c_int64(int(H)),
                                                        C.c_float(max_g), C.c_float(max_h), C.c_float(lower), C.c_float(upper),
                                                        None if mask is None else mask.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(out)))
        return json.loads(out.value.decode())

    def booster_predict_kernel_ms(self, bh, dh, repeats=5):
        ms = C.c_float()
        self._check(self.lib.XGB200BoosterPredictKernelMs(bh, dh, C.c_int(repeats), C.byref(ms)))
        return float(ms.value)

    def booster_predict_plan(self, bh, dh, iteration_range=(0, 0)):
        """The predictor's plan for this matrix and rounds, as a dict (include/b200xgb.h XGB200BoosterPredictPlan)."""
        out = C.c_char_p()
        self._check(self.lib.XGB200BoosterPredictPlan(bh, dh, C.c_int(iteration_range[0]), C.c_int(iteration_range[1]), C.byref(out)))
        return json.loads(out.value.decode())

    def booster_eval_container_metrics(self, bh, dh, names, output_margin):
        """Raw results of the container's own metrics on this matrix, int64[8 + 64 * 64]
        (include/b200xgb.h XGB200BoosterEvalContainerMetrics)."""
        arr = (C.c_char_p * len(names))(*[n.encode("utf-8") for n in names])
        out = np.zeros(8 + 64 * 64, np.int64)
        self._check(self.lib.XGB200BoosterEvalContainerMetrics(bh, dh, arr, c_bst_ulong(len(names)), C.c_int(1 if output_margin else 0),
                                                               out.ctypes.data_as(C.POINTER(C.c_longlong))))
        return out

    def booster_cached_margin(self, bh, dh, K):
        n = self.dmatrix_num_row(dh)
        out = np.zeros((n, K), np.float32)
        self._check(self.lib.XGB200BoosterGetCachedMargin(bh, dh, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def booster_compute_gradient(self, bh, dh, margin, round=0):
        """The configured objective's (g, h) at the given margins with round `round`'s row sample: float32 (n, K, 2)
        (include/b200xgb.h XGB200BoosterComputeGradient)."""
        n = self.dmatrix_num_row(dh)
        margin = np.ascontiguousarray(margin, np.float32).reshape(n, -1)
        out = np.zeros((n, margin.shape[1], 2), np.float32)
        self._check(self.lib.XGB200BoosterComputeGradient(bh, dh, margin.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(int(round)),
                                                          out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def booster_tree_weights(self, bh):
        """Each tree's weight in model order (booster=dart: weight_drop; all 1 for gbtree)."""
        n = c_bst_ulong()
        self._check(self.lib.XGB200BoosterGetTreeWeights(bh, C.byref(n), None))
        out = np.zeros(n.value, np.float32)
        self._check(self.lib.XGB200BoosterGetTreeWeights(bh, C.byref(n), out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def booster_refresh_sums(self, bh):
        """process_type=update: the int64 (G_q, H_q) of every node of the trees being updated, shape (nodes, 2), in the node order
        of the trees before the update (include/b200xgb.h XGB200BoosterGetRefreshSums)."""
        n = c_bst_ulong()
        self._check(self.lib.XGB200BoosterGetRefreshSums(bh, C.byref(n), None))
        out = np.zeros(n.value, np.int64)
        self._check(self.lib.XGB200BoosterGetRefreshSums(bh, C.byref(n), out.ctypes.data_as(C.POINTER(C.c_longlong))))
        return out.reshape(-1, 2)

    def timer_start(self):
        self._check(self.lib.XGB200TimerStart())

    def timer_stop(self):
        ms = C.c_float()
        self._check(self.lib.XGB200TimerStop(C.byref(ms)))
        return float(ms.value)

    def booster_set_profile(self, bh, enable):
        self._check(self.lib.XGB200BoosterSetProfile(bh, C.c_int(1 if enable else 0)))

    def booster_get_profile(self, bh):
        out = C.c_char_p()
        self._check(self.lib.XGB200BoosterGetProfile(bh, C.byref(out)))
        return json.loads(out.value.decode())

    def launch_count(self):
        out = C.c_longlong()
        self._check(self.lib.XGB200LaunchCount(C.byref(out)))
        return int(out.value)

    def synchronize(self):
        self._check(self.lib.XGB200Synchronize())


_BACKEND = None


def get_backend():
    """The process-wide backend. Tests may replace `_BACKEND` (e.g. with the oracle-backed engine in tests/)."""
    global _BACKEND
    if _BACKEND is None:
        _BACKEND = CudaBackend()
    return _BACKEND
