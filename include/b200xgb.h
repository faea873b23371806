/*
 * b200xgb.h -- C ABI of libb200xgb.so: an H100-native (sm_90a) gradient-boosted-tree trainer / predictor.
 *
 * DROP-IN BOUNDARY.  The SageMaker XGBoost container (aws/sagemaker-xgboost-container) never calls C directly:
 * it imports the `xgboost` Python package, which binds libxgboost's C API (include/xgboost/c_api.h of
 * xgboost==3.0.5, docker/3.0-5/base/Dockerfile.cpu:33) with ctypes.  The entry points below are the subset of
 * that C API the container's hot path reaches, with the same names, argument meaning, ownership and error
 * convention, so the same ctypes binding works against this library (see INTEGRATION.md).  Each declaration
 * cites the reference call site (file:line under src/sagemaker_xgboost_container of the reference container) that
 * reaches it through the Python package.
 *
 * Conventions (identical to libxgboost):
 *   - every function returns 0 on success, -1 on failure; XGBGetLastError() returns the thread-local message;
 *   - handles are opaque; out-pointers (strings, float arrays, shapes) are owned by the handle / a thread-local
 *     buffer and stay valid until the next call on the same handle from the same thread;
 *   - all buffers passed in are HOST memory; the library copies them to the GPU.  There is NO CPU fallback:
 *     without a CUDA device every call that needs one fails with an error.
 */
#ifndef B200XGB_H_
#define B200XGB_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define XGB_DLL __attribute__((visibility("default")))
#else
#define XGB_DLL
#endif

typedef void* DMatrixHandle;
typedef void* BoosterHandle;
typedef uint64_t bst_ulong;

XGB_DLL const char* XGBGetLastError(void);
/* fills major/minor/patch of the xgboost API level this library mirrors (3.0.5) */
XGB_DLL void XGBoostVersion(int* major, int* minor, int* patch);
/* JSON describing the build: {"USE_CUDA": true, "arch": "sm_90a", ...} */
XGB_DLL int XGBuildInfo(const char** out);

/* ---- DMatrix: data_utils.py:309-313,361,384,453 ; encoder.py:52,76,87,98 ; serve_utils.py:137,205 ---------- */
/* dense row-major float matrix, `missing` marks absent values (NaN is always missing) */
/* upstream's Python package passes ndarray inputs as `__array_interface__` JSON ({"data":[ptr,ro],"shape":[n,m],"typestr":"<f4"}),
 * config {"missing": NaN, "nthread": 0}; data_utils.py:384 (Parquet -> numpy), encoder.py:52 (CSV payload) reach it */
XGB_DLL int XGDMatrixCreateFromDense(const char* data, const char* config, DMatrixHandle* out);
/* labels / weights / base_margin from an array interface (DMatrix(label=...), data_utils.py:384); "group" (query group sizes) and
 * "qid" (one query id per row, non-decreasing; groups are its runs) from DMatrix(group=...) / DMatrix(qid=...) / set_info.  A 2-D
 * (n, T) "label" with T > 1 is a multi-target label (its rows must be the matrix's rows); GetFloatInfo returns it flat, row-major */
XGB_DLL int XGDMatrixSetInfoFromInterface(DMatrixHandle handle, const char* field, const char* data);
/* {"uri": "<path>?format=csv&label_column=0[&weight_column=1][&delimiter=,]" | "<path>?format=libsvm"}: data_utils.py:309-313,361;
 * a directory means every regular file in it (data_utils.py:520-545); CSV text is parsed on the device; libsvm qid:<id> tokens
 * become the query groups (the runs of equal consecutive qid over the files in order) */
XGB_DLL int XGDMatrixCreateFromURI(const char* config, DMatrixHandle* out);
XGB_DLL int XGDMatrixCreateFromMat(const float* data, bst_ulong nrow, bst_ulong ncol, float missing, DMatrixHandle* out);
/* CSR; num_col = 0 means "infer from the indices" (libsvm loader: indices kept as-is, data_utils.py:348-365) */
XGB_DLL int XGDMatrixCreateFromCSREx(const size_t* indptr, const unsigned* indices, const float* data, size_t nindptr,
                             size_t nelem, size_t num_col, DMatrixHandle* out);
/* device-resident input (what the reference's GPU path feeds through cupy/cudf, distributed_gpu/dask_data_utils.py:71-78):
 * `data` is a JSON __cuda_array_interface__ {"data":[ptr,ro],"shape":[n,F],"typestr":"<f4"[,"strides":null]},
 * config JSON {"missing": NaN} */
XGB_DLL int XGDMatrixCreateFromCudaArrayInterface(const char* data, const char* config, DMatrixHandle* out);

/* ---- QuantileDMatrix from a data iterator.  The names follow upstream's c_api.h; the signatures are recalled from its 3.0
 * release and were not checked against its source.  A proxy DMatrix carries one batch: next(iter) sets its data with one of
 * the XGProxyDMatrixSetData* calls and its meta information with XGDMatrixSetInfoFromInterface (label, weight, base_margin,
 * qid, label_lower_bound, label_upper_bound), then returns 1 (a batch), 0 (the end) or -1 (an error).  The batch's buffers must
 * stay valid until the next call of next or reset.  The proxy serves no other DMatrix call. */
typedef void* DataIterHandle;
typedef int XGDMatrixCallbackNext(DataIterHandle iter);
typedef void DataIterResetCallback(DataIterHandle iter);
XGB_DLL int XGProxyDMatrixCreate(DMatrixHandle* out);
/* host array interface JSON, 2-D, C-contiguous, any numeric typestr (other than <f4 converted to float32) */
XGB_DLL int XGProxyDMatrixSetDataDense(DMatrixHandle handle, const char* data);
/* __cuda_array_interface__ JSON, float32, C-contiguous: read in place (after a device synchronise) unless `missing` is not NaN */
XGB_DLL int XGProxyDMatrixSetDataCudaArrayInterface(DMatrixHandle handle, const char* data);
/* host CSR as three array interfaces: indptr (<u8 / <i8), indices (<u4 / <i4), data (<f4); ncol 0 = from the indices.  Absent
 * entries are missing; `missing` does not apply to the stored values (as XGDMatrixCreateFromCSREx) */
XGB_DLL int XGProxyDMatrixSetDataCSR(DMatrixHandle handle, const char* indptr, const char* indices, const char* data, bst_ulong ncol);
/* reset / next iterate the batches twice (once when there is only one batch).  config JSON: {"missing": float, "max_bin": int}
 * (defaults NaN and 256).  ref (a DMatrixHandle, or NULL): take its cuts and max_bin.  One process only: raises under a
 * communicator with world_size > 1. */
XGB_DLL int XGQuantileDMatrixCreateFromCallback(DataIterHandle iter, DMatrixHandle proxy, DataIterHandle ref, DataIterResetCallback* reset,
                                                XGDMatrixCallbackNext* next, const char* config, DMatrixHandle* out);

XGB_DLL int XGDMatrixFree(DMatrixHandle handle);
XGB_DLL int XGDMatrixNumRow(DMatrixHandle handle, bst_ulong* out);                                   /* train.py:339-342 */
XGB_DLL int XGDMatrixNumCol(DMatrixHandle handle, bst_ulong* out);
/* field: "label" | "weight" | "base_margin" */
XGB_DLL int XGDMatrixSetFloatInfo(DMatrixHandle handle, const char* field, const float* array, bst_ulong len);
XGB_DLL int XGDMatrixGetFloatInfo(DMatrixHandle handle, const char* field, bst_ulong* out_len, const float** out_dptr); /* train.py:394-396 get_label */
XGB_DLL int XGDMatrixSliceDMatrix(DMatrixHandle handle, const int* idxset, bst_ulong len, DMatrixHandle* out);          /* train.py:410-411 */
/* DMatrix.slice(rindex, allow_groups): with query groups, allow_groups != 0 and idxset listing whole groups (the slice keeps them) */
XGB_DLL int XGDMatrixSliceDMatrixEx(DMatrixHandle handle, const int* idxset, bst_ulong len, DMatrixHandle* out, int allow_groups);
/* query groups (rank:pairwise / rank:ndcg / rank:map, the ndcg / map metrics; DMatrix.set_group / set_uint_info / get_uint_info /
 * get_group): field "group_ptr" (len = groups + 1, from 0 to num_row) or "group" (the sizes); Get returns "group_ptr", empty
 * without groups */
XGB_DLL int XGDMatrixSetUIntInfo(DMatrixHandle handle, const char* field, const unsigned* array, bst_ulong len);
XGB_DLL int XGDMatrixGetUIntInfo(DMatrixHandle handle, const char* field, bst_ulong* out_len, const unsigned** out_dptr);
XGB_DLL int XGDMatrixSetGroup(DMatrixHandle handle, const unsigned* group, bst_ulong len);
/* field: "feature_name" | "feature_type" */
XGB_DLL int XGDMatrixSetStrFeatureInfo(DMatrixHandle handle, const char* field, const char** features, bst_ulong size);
XGB_DLL int XGDMatrixGetStrFeatureInfo(DMatrixHandle handle, const char* field, bst_ulong* size, const char*** out_features);

/* ---- Booster: train.py:367-376,432-442 (xgb.train) ; checkpointing.py:74 ------------------------------------ */
XGB_DLL int XGBoosterCreate(const DMatrixHandle dmats[], bst_ulong len, BoosterHandle* out);
XGB_DLL int XGBoosterFree(BoosterHandle handle);
XGB_DLL int XGBoosterSetParam(BoosterHandle handle, const char* name, const char* value);
/* one boosting round of the configured objective on dtrain (the hot path) */
XGB_DLL int XGBoosterUpdateOneIter(BoosterHandle handle, int iter, DMatrixHandle dtrain);
/* custom objective: not implemented on the device path, returns -1 */
XGB_DLL int XGBoosterBoostOneIter(BoosterHandle handle, DMatrixHandle dtrain, float* grad, float* hess, bst_ulong len);
/* "[iter]\t<name>-<metric>:<value>..." -- callback.py:85 EvaluationMonitor parses this */
XGB_DLL int XGBoosterEvalOneIter(BoosterHandle handle, int iter, DMatrixHandle dmats[], const char* evnames[], bst_ulong len,
                         const char** out_result);
/* config JSON: {"type": 0 value | 1 margin | 6 leaf, "training": bool, "iteration_begin": int,
 *               "iteration_end": int, "strict_shape": bool}
 * serve_utils.py:244-250, serving.py:98, handler_service.py:73, train.py:445 */
XGB_DLL int XGBoosterPredictFromDMatrix(BoosterHandle handle, DMatrixHandle dmat, const char* config,
                                bst_ulong const** out_shape, bst_ulong* out_dim, float const** out_result);
/* file name extension picks the format: .json -> JSON text, anything else (incl. none) -> UBJSON  (train.py:480) */
XGB_DLL int XGBoosterSaveModel(BoosterHandle handle, const char* fname);
XGB_DLL int XGBoosterLoadModel(BoosterHandle handle, const char* fname);                              /* serve_utils.py:184-185 */
/* config JSON: {"format": "ubj" | "json"} */
XGB_DLL int XGBoosterSaveModelToBuffer(BoosterHandle handle, const char* config, bst_ulong* out_len, const char** out_dptr);
XGB_DLL int XGBoosterLoadModelFromBuffer(BoosterHandle handle, const void* buf, bst_ulong len);
/* model + configuration, used for pickling (serve_utils.py:180-182 pickle.load of a Booster) */
XGB_DLL int XGBoosterSerializeToBuffer(BoosterHandle handle, bst_ulong* out_len, const char** out_dptr);
XGB_DLL int XGBoosterUnserializeFromBuffer(BoosterHandle handle, const void* buf, bst_ulong len);
XGB_DLL int XGBoosterSaveJsonConfig(BoosterHandle handle, bst_ulong* out_len, const char** out_str);  /* serve.py:85-88 */
XGB_DLL int XGBoosterLoadJsonConfig(BoosterHandle handle, const char* config);
XGB_DLL int XGBoosterGetNumFeature(BoosterHandle handle, bst_ulong* out);
XGB_DLL int XGBoosterBoostedRounds(BoosterHandle handle, int* out);
XGB_DLL int XGBoosterSlice(BoosterHandle handle, int begin_layer, int end_layer, int step, BoosterHandle* out); /* EarlyStopping save_best */
XGB_DLL int XGBoosterGetAttr(BoosterHandle handle, const char* key, const char** out, int* success);  /* best_iteration */
XGB_DLL int XGBoosterSetAttr(BoosterHandle handle, const char* key, const char* value);               /* value NULL deletes */
XGB_DLL int XGBoosterGetAttrNames(BoosterHandle handle, bst_ulong* out_len, const char*** out);
XGB_DLL int XGBoosterSetStrFeatureInfo(BoosterHandle handle, const char* field, const char** features, bst_ulong size);
XGB_DLL int XGBoosterGetStrFeatureInfo(BoosterHandle handle, const char* field, bst_ulong* len, const char*** out_features);

/* ---- collective: distributed.py:119-136,219-220,238-243 (xgboost.collective) --------------------------------- */
/* config JSON: {"nccl_unique_id": "<hex, 128 bytes>", "rank": r, "world_size": w}; the id comes from
 * XGCommunicatorGetUniqueId on rank 0 and is shipped by the Python-side bootstrap (tracker / torch.distributed). */
XGB_DLL int XGCommunicatorInit(const char* config);
/* broadcast of a host buffer from `root` (distributed.py:119-136 via xgboost.collective.broadcast) */
XGB_DLL int XGCommunicatorBroadcast(void* send_receive_buffer, size_t size, int root);
XGB_DLL int XGCommunicatorFinalize(void);
XGB_DLL int XGCommunicatorGetRank(void);
XGB_DLL int XGCommunicatorGetWorldSize(void);
XGB_DLL int XGCommunicatorGetUniqueId(const char** out_hex);

/* ---- build-specific introspection (no libxgboost counterpart; used by tests/ and bench.py) -------------------- */
/* cuts as an explicit artefact shared with the oracle: ptrs[F+1], vals[ptrs[F]], mins[F] */
XGB_DLL int XGB200DMatrixGetCuts(DMatrixHandle handle, int max_bin, bst_ulong* n_ptrs, const int** ptrs, bst_ulong* n_vals,
                         const float** vals, const float** mins, int* has_missing);
XGB_DLL int XGB200DMatrixSetCuts(DMatrixHandle handle, const int* ptrs, bst_ulong n_ptrs, const float* vals, const float* mins);
/* Serving input path (SURVEY.md 8f-1): a CSV request body parsed on the device into the DMatrix.  Replaces the Python
 * split + np.array(...).astype(float) of encoder.csv_to_dmatrix (encoder.py:35-52, reached from serve_utils.py:121-131).
 * `text` is the stripped payload ('\n' between rows, `delimiter` between fields, empty field = NaN).  *status: 0 = parsed,
 * 1 = rows of different lengths, 2 = a field the exact device fast path cannot decide (caller parses on the host);
 * *out is NULL unless *status == 0. */
XGB_DLL int XGB200DMatrixCreateFromCSV(const char* text, bst_ulong len, char delimiter, int* status, DMatrixHandle* out);
/* Training loaders to the device (SURVEY.md 8f-2): the text of a CSV channel ("<dir>?format=csv&label_column=0[&weight_column=1]",
 * data_utils.py:289-318) parsed on the GPU; label_column / weight_column (-1 = none) become the "label" / "weight" float
 * info, the other columns the feature matrix.  Same status convention as XGB200DMatrixCreateFromCSV. */
XGB_DLL int XGB200DMatrixCreateFromCSVEx(const char* text, bst_ulong len, char delimiter, int label_column, int weight_column,
                             int* status, DMatrixHandle* out);
/* 1 when the per-level histogram all-reduce runs as the NVLink peer-memory kernel (nvlink.cu), 0 when it goes through NCCL */
/* A libsvm request body ("label idx:val ..." lines, already stripped) parsed on the device into a dense matrix.
 * whitespace_mode 0 / absent NaN = serve_utils._get_sparse_matrix_from_libsvm + xgb.DMatrix(csr) (algorithm_mode/serve_utils.py:94-118,
 * 132-137: tokens split on ' ', entries a line does not list are missing); whitespace_mode 1 / absent 0 = encoder.libsvm_to_dmatrix
 * (encoder.py:54-86: split on any whitespace, dense zeros).  Indices shift to 0-based when the smallest one is >= 1, as both do.
 * *status: 0 ok; 2 = the body holds something the Python routes treat specially (non-digit index, literal outside the exact
 * fast path, repeated index in a line, trailing empty lines ...): take the host route; 3 = no entry at all (ditto). */
XGB_DLL int XGB200DMatrixCreateFromLibsvmText(const char* text, bst_ulong len, int whitespace_mode, float absent, int* status, DMatrixHandle* out);
/* A recordio-protobuf body (application/x-recordio-protobuf: the whole request, or the concatenated files of a training channel)
 * decoded on the device into the DMatrix that xgb.DMatrix(features, label=labels) holds for the reference's
 * `features, labels = read_recordio_protobuf(buf)`: encoder.recordio_protobuf_to_dmatrix (serve_utils.py:144-145) and
 * data_utils.get_recordio_protobuf_dmatrix (data_utils.py:450-453).  features["values"] of every record is a row (dense, or sparse
 * when its tensor has keys), label["values"] values are concatenated into the "label" info.  *status: 0 = decoded (*out set);
 * 1 = the reference raises ValueError for this body (bad magic, truncated record, rows of different widths, no record): the
 * message is what XGBGetLastError() returns; 2 = the body holds an encoding the device path does not decide (unpacked or
 * repeated fields, merged messages, a repeated "values" key, malformed protobuf ...): decode it on the host.  The return value
 * is non-zero only for a failure of the library itself. */
XGB_DLL int XGB200DMatrixCreateFromRecordIO(const char* buf, bst_ulong len, int* status, DMatrixHandle* out);
XGB_DLL int XGB200CommPeerReduceActive(void);
/* Columnar training input without a dense float32 matrix on the host (Parquet through pyarrow, pandas frames): `ncols` host
 * buffers of `nrow` items each, col_types[c] in {0 f32, 1 f64, 2 i32, 3 i64, 4 u8, 5 i8, 6 i16, 7 u16, 8 u32, 9 u64, 10 bool};
 * the buffers cross PCIe as they are and are converted (round to nearest, like numpy's astype(float32)) and transposed into
 * the row-major matrix on the device (ingest.cu).  label_column / weight_column (-1 = none) become the label / weight info.
 * Replaces the host copies of data_utils.get_parquet_dmatrix (data_utils.py:368-390: read_table -> to_pandas -> to_numpy ->
 * data[:, 1:]) in front of XGDMatrixCreateFromMat. */
XGB_DLL int XGB200DMatrixCreateFromColumns(const void* const* cols, const int* col_types, int ncols, bst_ulong nrow, int label_column,
                                   int weight_column, DMatrixHandle* out);
/* the float32 feature matrix as the engine holds it (row-major n x F, NaN = missing), for bit-exact checks of the input paths */
XGB_DLL int XGB200DMatrixGetRaw(DMatrixHandle handle, float* out_row_major);
/* device bytes the engine holds in its buffers now (*live) and at most since the last reset (*peak); reset_peak != 0 first
 * sets the peak to the live bytes.  Allocations outside the engine's buffer type (a 4 KB peer-exchange word) are not counted. */
XGB_DLL int XGB200DeviceMemory(bst_ulong* live, bst_ulong* peak, int reset_peak);
/* binned feature blocks back on the host in plain row-major n x F order (for bit-exact checks of the binning kernel) */
XGB_DLL int XGB200DMatrixGetBins(DMatrixHandle handle, int max_bin, uint8_t* out_row_major);
/* the two other binned copies the kernels read: the 128 B line-aligned row copy (built when the main block is 96 B wide;
 * *out_aligned_stride = 128 and out_aligned gets n x 128 bytes, else *out_aligned_stride = 0 and out_aligned is not written)
 * and the column-major copy (out_col: F x n).  Any pointer may be NULL. */
XGB_DLL int XGB200DMatrixGetBinCopies(DMatrixHandle handle, int max_bin, int* out_aligned_stride, uint8_t* out_aligned, uint8_t* out_col);
/* the multi-GPU cut recipe run on one GPU: rows [row_bounds[r], row_bounds[r + 1]) of `handle` (r < n_ranges, covering all rows)
 * stand for rank r's shard; each gets the capped per-rank summary, the summaries are merged in rank order and the cuts derived
 * as every rank would.  Does not touch the matrix's own cuts.  out_ptrs: F+1, out_vals: capacity F x 256, out_mins: F. */
XGB_DLL int XGB200DMatrixRankCuts(DMatrixHandle handle, int max_bin, const int64_t* row_bounds, int n_ranges, int* out_ptrs,
                          float* out_vals, float* out_mins);
/* the alpha-quantile of each segment with the select kernels of reg:absoluteerror's leaf refresh: values[i] belongs to segment
 * segments[i] (in [0, n_segments), or -1 = left out; NULL = every value in segment 0).  Without weights, upstream's Quantile
 * (interpolated between order statistics); with weights (rows of weight 0 left out), the first value in sorted order whose
 * cumulative weight reaches alpha * total, the weights counted on the training histograms' fixed-point grid for n rows.
 * -0.0 counts as +0.0; a NaN value is an error.  out: n_segments floats, NaN for a segment without values. */
XGB_DLL int XGB200SegmentedQuantile(const float* values, const int32_t* segments, const float* weights, bst_ulong n, int n_segments,
                                    float alpha, float* out);
/* sampling_method=gradient_based on caller-given pairs (gpair: n x 2 floats (g, h)), with the select and sampling kernels of
 * training: rag = sqrtf(g^2 + 0.1 h^2), k = max(1, (int64)(float(n) * subsample)) and the threshold u with
 * sum_i min(1, rag_i / u) = k (0: every row is kept as it is, when k >= the rows with rag > 0); then row i with p = rag_i / u < 1
 * and a finite rag is kept when rng_uniform(seed, stream, i) < p, as (g / p, h / p), and zeroed otherwise.
 * *out_threshold = u; out_gpair: n x 2 floats, the sampled pairs. */
XGB_DLL int XGB200GradientBasedSample(const float* gpair, bst_ulong n, float subsample, unsigned seed, uint64_t stream,
                                      float* out_threshold, float* out_gpair);
/* flat tree arrays of the model; any pointer may be NULL. tree_offset has num_trees+1 entries. */
/* num_class: the outputs per row (the class count of multi:*, len(quantile_alpha) of reg:quantileerror, else 1) */
XGB_DLL int XGB200BoosterModelShape(BoosterHandle handle, bst_ulong* num_trees, bst_ulong* num_nodes, float* base_score, int* num_class);
XGB_DLL int XGB200BoosterExportModel(BoosterHandle handle, int64_t* tree_offset, int32_t* tree_info, int32_t* left, int32_t* right,
                             int32_t* parent, int32_t* split_index, int32_t* split_bin, uint8_t* default_left,
                             float* split_cond, float* base_weight, float* loss_chg, float* sum_hess);
/* root histogram of `dmat` for host gradient pairs (n x 2 floats): out_hist is int64 [F][256][2] fixed point,
 * scales[4] = {sg, sh, 1/sg, 1/sh}; the kernel is launched `repeats` times and its mean device time returned. */
XGB_DLL int XGB200BuildRootHistogram(BoosterHandle handle, DMatrixHandle dmat, const float* gpair, int repeats,
                             int64_t* out_hist, float* scales, float* out_ms);
/* same with a kernel choice and an optional row subset: mode 0 = production choice (TMA-staged root kernel), 1 = gather
 * kernel, 2 = G-only TMA root kernel (constant-hessian fast path: the H plane of out_hist stays zero).  With row_ids
 * (n_ids entries, ascending or not) the histogram covers that subset and gpair is given by POSITION (gpair[i] belongs to
 * row row_ids[i]) -- the deeper tree levels' access pattern.  Added to the mode: 4 = the tail bytes come from where the
 * training path takes them (by position for a 4-wide tail the line-aligned row copy does not hold; that copy's line when it
 * does), 8 = G-only payload of the constant-hessian levels (only g of gpair is used, h == 1.0f for every row).
 * out_kernel: name of the kernel variant that ran. */
XGB_DLL int XGB200BuildHistogramEx(BoosterHandle handle, DMatrixHandle dmat, const float* gpair, int repeats, int mode,
                             const unsigned* row_ids, bst_ulong n_ids, int64_t* out_hist, float* scales, float* out_ms,
                             const char** out_kernel);
/* split evaluation of one root, with the training path's kernels and arguments: `hist` is int64 [F][256][2] fixed point (g, h)
 * on the grid launch_scales derives from max_g = max|g| and max_h = max h for the row count of `dmat`, which supplies the layout
 * and the cuts (XGB200DMatrixSetCuts); (G, H) are the node totals in grid units, [lower, upper] the root's weight bounds (only
 * read under monotone constraints), feat_mask (F bytes, 1 = usable; NULL = all) the tree's column set.  Runs init_tree,
 * eval_kernel at level 0 and the grow_policy's expansion.  *out_json: {"scales": [4], "root_gain", "weight", "best_group":
 * [per candidate block], "best", "n_nodes", "expanded", "tree": {the arrays of nodes 0 .. n_nodes-1}, "children": [{"G", "H",
 * "lower", "upper"}]}; a candidate is {"loss_chg", "feature", "bin", "dleft", "ord", "GL", "HL"}; every float is its uint32 bits. */
XGB_DLL int XGB200BoosterEvalRootSplit(BoosterHandle handle, DMatrixHandle dmat, const int64_t* hist, int64_t G, int64_t H, float max_g,
                               float max_h, float lower, float upper, const uint8_t* feat_mask, const char** out_json);
/* mean device time (CUDA events) of the predictor kernel alone over `repeats` launches on `dmat` */
XGB_DLL int XGB200BoosterPredictKernelMs(BoosterHandle handle, DMatrixHandle dmat, int repeats, float* out_ms);
/* the predictor's plan for `dmat` and the rounds [iter_begin, iter_end) (iter_end == 0: all), without running it: JSON
 * {"kernel": "predict_tiled_kernel" | "predict_kernel", "reason" (why thread-per-row), "has_nan", "tree_begin", "tree_end",
 * "pitch", "chunks": [{"begin","end","node_bytes","rows","threads","smem"}]} (see csrc/predict_plan.h) */
XGB_DLL int XGB200BoosterPredictPlan(BoosterHandle handle, DMatrixHandle dmat, int iter_begin, int iter_end, const char** out_json);
/* the container's own metrics (sagemaker_xgboost_container custom_metrics: accuracy, balanced_accuracy, f1, f1_binary,
 * f1_macro, precision[_macro|_micro], recall[_macro|_micro], mse, rmse, mae, r2) on `dmat`, from the prediction cache: the
 * raw results out[8 + 64 * 64] (csrc/container_metrics.h): out[0] bits decided (1 confusion counts, 2 regression sums, 4 the
 * label sums of r2), out[1] rows, out[2] predicted classes P, out[3] label bound L = 64, out[4..8) float32 bits of
 * sum (y-p)^2, sum |y-p|, sum y, sum (y-mean)^2 in numpy's pairwise order, out[8..] counts [L][P].  output_margin: the
 * metric reads the margins (feval=) rather than predict()'s values */
XGB_DLL int XGB200BoosterEvalContainerMetrics(BoosterHandle handle, DMatrixHandle dmat, const char** names, bst_ulong len, int output_margin,
                                              long long* out);
/* raw margins of the prediction cache the trainer keeps for `dmat` (n x outputs per row), brought up to date first */
XGB_DLL int XGB200BoosterGetCachedMargin(BoosterHandle handle, DMatrixHandle dmat, float* out);
/* the weight of every tree in model order (booster=dart: weight_drop; 1 for gbtree); out may be NULL to query the length */
XGB_DLL int XGB200BoosterGetTreeWeights(BoosterHandle handle, bst_ulong* len, float* out);
/* process_type=update: the exact fixed-point (G_q, H_q) sums of every node of every tree being updated, in the node order of the
 * trees as they were before the update (trees one after another), 2 int64 per node; the nodes of layers not yet updated are 0.
 * len = 0 before the first update round.  out may be NULL to query len. */
XGB_DLL int XGB200BoosterGetRefreshSums(BoosterHandle handle, bst_ulong* len, long long* out);
/* the configured objective's gradient pairs on `dmat` at the given margins (n x outputs per row, host), with the row sample of boosting
 * round `round` (subsample < 1: unsampled rows are (0, 0)); out_gpair: n x outputs x 2 floats (g, h).  Under
 * sampling_method=gradient_based that sample is the one tree 0 of each class takes: each class's own threshold over these
 * pairs, the draws of the round's uniform sample, kept rows scaled by 1 / p (XGB200GradientBasedSample). */
XGB_DLL int XGB200BoosterComputeGradient(BoosterHandle handle, DMatrixHandle dmat, const float* margin, int round, float* out_gpair);
/* CUDA-event stopwatch on the engine's stream: Start records an event, Stop records another, waits, returns ms */
XGB_DLL int XGB200TimerStart(void);
XGB_DLL int XGB200TimerStop(float* out_ms);
/* per-kernel profile of the tree builder (CUDA events around each launch group of the rounds run while enabled): enable,
 * run rounds, then read {"root_hist_ms","root_hist_launches","root_hist_rows","deep_hist_ms","deep_hist_launches",
 * "deep_hist_rows","part_ms","part_launches","part_rows" (rows of split nodes),"part_rows_written","part_row_bytes_in_root",
 * "part_row_bytes_in","part_row_bytes_out" (the partition's bytes per row read at the root level, read at deeper levels and
 * written),"margin_ms","margin_launches","margin_rows"} */
XGB_DLL int XGB200BoosterSetProfile(BoosterHandle handle, int enable);
XGB_DLL int XGB200BoosterGetProfile(BoosterHandle handle, const char** out_json);
/* number of CUDA kernels this library has launched so far in this process */
XGB_DLL int XGB200LaunchCount(long long* out);
/* wait for all device work queued by this library */
XGB_DLL int XGB200Synchronize(void);
/* Host-only converter: a pre-JSON binary model (Booster.save_model of xgboost < 2, optionally behind the "CONFIG-offset:"
 * prefix of a pickled 1.x Booster) -> the UBJSON model document XGBoosterLoadModelFromBuffer reads.  The loaders call the
 * same code internally (legacy_io.cc); exported so that old model archives can be migrated, and checked, without a GPU.
 * Replaces: libxgboost's LearnerIO::LoadModel legacy branch behind serve_utils.get_loaded_booster
 * (algorithm_mode/serve_utils.py:171-197; fixtures test/resources/models/{saved_booster,pickled_model}).
 * *out is a thread-local buffer, valid until the next call of this function on the same thread. */
XGB_DLL int XGB200LegacyModelToUBJ(const void* buf, bst_ulong len, bst_ulong* out_len, const char** out);

#ifdef __cplusplus
}
#endif
#endif /* B200XGB_H_ */
