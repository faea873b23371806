// booster.cu -- DMatrix / Booster implementation: the round loop of `xgb.train` (Booster.update) on the device.
// Reference call sites served: algorithm_mode/train.py:367-376,432-442 (xgb.train), serve_utils.py:244-250
// (Booster.predict), data_utils.py:309-313,361,384 (DMatrix construction).  Upstream behaviour restated:
// src/learner.cc (UpdateOneIter, EvalOneIter, base_score), src/gbm/gbtree.cc (DoBoost, one tree per class).
#include "booster.h"
#include <algorithm>
#include <atomic>
#include <cctype>
#include <climits>
#include <cmath>
#include <cstring>
#include "comm.h"
#include "multi_target.h"
#include "rng.h"

namespace b200 {

long long g_kernel_launches = 0;

// ---------------------------------------------------------------------------------------------
// process-wide device context
// ---------------------------------------------------------------------------------------------
namespace {
struct DeviceCtx {
  cudaStream_t stream = nullptr; int num_sms = 0; bool ok = false; std::string why;
  DeviceCtx() {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) { why = std::string("no CUDA device available (") + cudaGetErrorString(e) + ")"; cudaGetLastError(); return; }
    int dev = 0;
    if (const char* lr = getenv("LOCAL_RANK")) { dev = atoi(lr) % count; }
    if (const char* d = getenv("B200XGB_DEVICE")) { dev = atoi(d) % count; }
    if (cudaSetDevice(dev) != cudaSuccess) { why = "cudaSetDevice failed"; return; }
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) { why = "cudaStreamCreate failed"; return; }
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    ok = true;
  }
};
DeviceCtx& ctx() { static DeviceCtx c; if (!c.ok) throw Error("b200xgb: " + c.why + "; this library has no CPU fallback"); return c; }
std::atomic<uint64_t> g_uid{1};
}  // namespace

cudaStream_t engine_stream() { return ctx().stream; }
int engine_num_sms() { return ctx().num_sms; }

namespace {
std::atomic<int64_t> g_devmem_live{0}, g_devmem_peak{0};
}  // namespace
void devmem_note(int64_t delta) {
  const int64_t now = g_devmem_live.fetch_add(delta) + delta;
  int64_t peak = g_devmem_peak.load();
  while (now > peak && !g_devmem_peak.compare_exchange_weak(peak, now)) {}
}
void devmem_query(uint64_t* live, uint64_t* peak, bool reset_peak) {
  if (reset_peak) g_devmem_peak.store(g_devmem_live.load());
  if (live) *live = (uint64_t)g_devmem_live.load();
  if (peak) *peak = (uint64_t)g_devmem_peak.load();
}

// ---------------------------------------------------------------------------------------------
// DMatrix
// ---------------------------------------------------------------------------------------------
DMatrix::DMatrix() : uid(g_uid++) {}

void DMatrix::require_raw(const char* what) const {
  B200_CHECK(!quantile, std::string(what) + " is not supported on a QuantileDMatrix: it keeps only the binned features; build a DMatrix for it");
}

void DMatrix::finish_upload(float missing) {
  cudaStream_t s = engine_stream();
  const int64_t count = n * F;
  const bool use_missing = !std::isnan(missing);
  DevBuf<unsigned long long> cnt; cnt.alloc(1); cnt.zero(s);
  launch_count_nan(X.p, count, missing, use_missing ? 1 : 0, cnt.p, s);
  if (use_missing) launch_replace_missing(X.p, count, missing, s);
  unsigned long long c = 0;
  CUDA_OK(cudaMemcpyAsync(&c, cnt.p, 8, cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  has_missing = c > 0;
}

std::unique_ptr<DMatrix> DMatrix::from_dense(const float* data, int64_t nrow, int ncol, float missing) {
  B200_CHECK(nrow >= 0 && ncol >= 0, "DMatrix: negative shape");
  B200_CHECK(nrow < (int64_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  auto dm = std::make_unique<DMatrix>();
  dm->n = nrow; dm->F = ncol;
  cudaStream_t s = engine_stream();
  dm->X.alloc((size_t)nrow * ncol);
  if (nrow * ncol > 0) {
    CUDA_OK(cudaMemcpyAsync(dm->X.p, data, sizeof(float) * (size_t)nrow * ncol, cudaMemcpyHostToDevice, s));
  }
  dm->finish_upload(missing);
  return dm;
}

std::unique_ptr<DMatrix> DMatrix::from_device(const float* dptr, int64_t nrow, int ncol, float missing) {
  B200_CHECK(nrow >= 0 && ncol >= 0 && nrow < (int64_t)0x7fffffff, "DMatrix: bad shape");
  auto dm = std::make_unique<DMatrix>();
  dm->n = nrow; dm->F = ncol;
  cudaStream_t s = engine_stream();
  dm->X.alloc((size_t)nrow * ncol);
  CUDA_OK(cudaDeviceSynchronize());       // the producer (e.g. a torch stream) must be done before we read its buffer
  if (nrow * ncol > 0) CUDA_OK(cudaMemcpyAsync(dm->X.p, dptr, sizeof(float) * (size_t)nrow * ncol, cudaMemcpyDeviceToDevice, s));
  dm->finish_upload(missing);
  return dm;
}

// DMatrix::from_csr / from_columns: ingest.cu (device-side densify / column transpose, no dense host copy)

__global__ void gather_rows_kernel(const float* X, int F, const int* idx, int64_t len, float* out) {
  const int64_t total = len * F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / F; int f = (int)(i % F);
    out[i] = X[(int64_t)idx[r] * F + f];
  }
}

std::unique_ptr<DMatrix> DMatrix::slice(const int* idx, int64_t len, bool allow_groups) const {
  require_raw("DMatrix.slice (and xgb.cv, which slices its folds)");
  for (int64_t i = 0; i < len; ++i) B200_CHECK(idx[i] >= 0 && idx[i] < n, "DMatrix.slice: row index out of range");
  // with query groups: idx must list whole groups, each one's rows in order; the slice keeps those groups (and their weights)
  std::vector<unsigned> ptr; std::vector<int> groups;
  if (!group_ptr.empty()) {
    B200_CHECK(allow_groups, "DMatrix.slice: the matrix has query groups; slice it by whole groups with allow_groups=True");
    ptr.push_back(0);
    for (int64_t i = 0; i < len;) {
      const int g = (int)(std::upper_bound(group_ptr.begin(), group_ptr.end(), (unsigned)idx[i]) - group_ptr.begin()) - 1;
      const int64_t size = (int64_t)group_ptr[g + 1] - group_ptr[g];
      B200_CHECK(idx[i] == (int)group_ptr[g] && i + size <= len, "DMatrix.slice: with allow_groups=True the rows must be whole query groups");
      for (int64_t j = 0; j < size; ++j) B200_CHECK(idx[i + j] == (int)(group_ptr[g] + j), "DMatrix.slice: with allow_groups=True the rows must be whole query groups");
      groups.push_back(g); i += size; ptr.push_back((unsigned)i);
    }
  }
  auto dm = std::make_unique<DMatrix>();
  dm->n = len; dm->F = F; dm->has_missing = has_missing;
  dm->feature_names = feature_names; dm->feature_types = feature_types;
  cudaStream_t s = engine_stream();
  dm->X.alloc((size_t)len * F);
  if (len * F > 0) {
    DevBuf<int> didx; didx.alloc(len);
    CUDA_OK(cudaMemcpyAsync(didx.p, idx, sizeof(int) * len, cudaMemcpyHostToDevice, s));
    int grid = (int)std::min<int64_t>((len * F + 255) / 256, engine_num_sms() * 16);
    gather_rows_kernel<<<grid, 256, 0, s>>>(X.p, F, didx.p, len, dm->X.p); ++g_kernel_launches;
    CUDA_OK(cudaGetLastError());
    Comm::get().sync_stream(s);
  }
  auto take = [&](const std::vector<float>& src, size_t per_row) { std::vector<float> o; if (src.empty()) return o; o.resize(len * per_row);
    for (int64_t i = 0; i < len; ++i) for (size_t k = 0; k < per_row; ++k) o[i * per_row + k] = src[(size_t)idx[i] * per_row + k]; return o; };
  if (!labels.empty()) { auto v = take(labels, (size_t)label_cols); dm->set_label_matrix(v.data(), len, label_cols); }      // whole label rows
  if (!group_ptr.empty()) {
    dm->set_group_ptr(ptr);
    if (!weights.empty()) {
      B200_CHECK(weights.size() == group_ptr.size() - 1, "DMatrix.slice: a matrix with query groups needs one weight per group");
      std::vector<float> v; for (int g : groups) v.push_back(weights[g]);
      dm->set_float_info("weight", v.data(), v.size());
    }
  } else if (!weights.empty()) { auto v = take(weights, 1); dm->set_float_info("weight", v.data(), v.size()); }
  if (!label_lower.empty()) { auto v = take(label_lower, 1); dm->set_float_info("label_lower_bound", v.data(), v.size()); }
  if (!label_upper.empty()) { auto v = take(label_upper, 1); dm->set_float_info("label_upper_bound", v.data(), v.size()); }
  if (!base_margin.empty() && n > 0) { size_t per = base_margin.size() / n; auto v = take(base_margin, per); dm->set_float_info("base_margin", v.data(), v.size()); }
  return dm;
}

void DMatrix::set_float_info(const std::string& field, const float* v, size_t len) {
  cudaStream_t s = engine_stream();
  auto put = [&](std::vector<float>& h, DevBuf<float>& d) {
    h.assign(v, v + len); d.alloc(len);
    if (len) { CUDA_OK(cudaMemcpyAsync(d.p, h.data(), sizeof(float) * len, cudaMemcpyHostToDevice, s)); Comm::get().sync_stream(s); }
  };
  if (field == "label") { put(labels, d_labels); label_cols = 1; cox_order.valid = false; rank_groups.valid = false; container_sums.labels_valid = false; }
  else if (field == "label_lower_bound") put(label_lower, d_label_lower);      // survival:aft; the bins do not depend on them
  else if (field == "label_upper_bound") put(label_upper, d_label_upper);
  else if (field == "weight") {
    for (size_t i = 0; i < len; ++i) B200_CHECK(v[i] >= 0 && !std::isnan(v[i]), "Weights must be positive values.");
    B200_CHECK(!quantile || group_ptr.empty(), "weights together with query groups are not supported on a QuantileDMatrix");
    put(weights, d_weights);
    binned = binned && quantile;      // weighted quantiles depend on the weights; a QuantileDMatrix keeps the cuts it was built with
    rank_groups.valid = false;
  }
  else if (field == "base_margin") put(base_margin, d_base_margin);
  else throw Error("Unknown float field name: " + field);
}

void DMatrix::set_label_matrix(const float* v, int64_t rows, int64_t cols) {
  B200_CHECK(cols >= 1 && cols <= INT_MAX, "label: a 2-D label needs at least one column");
  B200_CHECK(rows == n, "label: the label has " + std::to_string(rows) + " rows but the DMatrix has " + std::to_string(n));
  set_float_info("label", v, (size_t)(rows * cols));
  label_cols = (int)cols;
}

void DMatrix::set_group_ptr(std::vector<unsigned> ptr) {
  B200_CHECK(!ptr.empty() && ptr[0] == 0, "group_ptr must start at 0");
  for (size_t g = 1; g < ptr.size(); ++g) B200_CHECK(ptr[g] >= ptr[g - 1], "group_ptr must not decrease");
  B200_CHECK((int64_t)ptr.back() == n, "the query groups cover " + std::to_string(ptr.back()) + " rows but the DMatrix has " + std::to_string(n) +
             " (group sizes must add up to num_row)");
  B200_CHECK(!quantile || weights.empty() || ptr.size() <= 1, "weights together with query groups are not supported on a QuantileDMatrix");
  group_ptr = ptr.size() > 1 ? std::move(ptr) : std::vector<unsigned>{};
  rank_groups.valid = false;
  binned = binned && (quantile || weights.empty());       // the sketch reads per-group weights row by row
}

void DMatrix::set_group_sizes(const unsigned* sizes, size_t len) {
  std::vector<unsigned> ptr{0};
  uint64_t at = 0;
  for (size_t g = 0; g < len; ++g) { at += sizes[g]; B200_CHECK(at <= (uint64_t)n, "the query group sizes add up to more than the " + std::to_string(n) + " rows of the DMatrix"); ptr.push_back((unsigned)at); }
  set_group_ptr(std::move(ptr));
}

void DMatrix::set_qid(const int64_t* qid, size_t len) {
  B200_CHECK((int64_t)len == n, "qid must have one entry per row (" + std::to_string(n) + " rows, " + std::to_string(len) + " qid)");
  std::vector<unsigned> ptr{0};
  for (size_t i = 1; i < len; ++i) {
    B200_CHECK(qid[i] >= qid[i - 1], "qid must be sorted in non-decreasing order (row " + std::to_string(i) + ": " + std::to_string(qid[i]) + " after " +
               std::to_string(qid[i - 1]) + ")");
    if (qid[i] != qid[i - 1]) ptr.push_back((unsigned)i);
  }
  if (len) ptr.push_back((unsigned)len);
  set_group_ptr(std::move(ptr));
}

const std::vector<float>& DMatrix::get_float_info(const std::string& field) const {
  if (field == "label") return labels;
  if (field == "weight") return weights;
  if (field == "base_margin") return base_margin;
  if (field == "label_lower_bound") return label_lower;
  if (field == "label_upper_bound") return label_upper;
  throw Error("Unknown float field name: " + field);
}

void DMatrix::bin_with_cuts() {
  alloc_bins();
  launch_bin(X.p, n, F, ngroups, tw, d_cut_ptrs.p, d_cut_vals.p, bins.p, bins_tail.p, engine_stream());
  finish_bins();
}

void DMatrix::alloc_bins() {
  cudaStream_t s = engine_stream();
  feature_layout(F, &ngroups, &tw, &ntail);
  ++binned_version;
  d_cut_ptrs.alloc(cuts.ptrs.size()); d_cut_vals.alloc(cuts.vals.size()); d_min_vals.alloc(cuts.mins.size());
  CUDA_OK(cudaMemcpyAsync(d_cut_ptrs.p, cuts.ptrs.data(), sizeof(int) * cuts.ptrs.size(), cudaMemcpyHostToDevice, s));
  if (!cuts.vals.empty()) CUDA_OK(cudaMemcpyAsync(d_cut_vals.p, cuts.vals.data(), sizeof(float) * cuts.vals.size(), cudaMemcpyHostToDevice, s));
  if (!cuts.mins.empty()) CUDA_OK(cudaMemcpyAsync(d_min_vals.p, cuts.mins.data(), sizeof(float) * cuts.mins.size(), cudaMemcpyHostToDevice, s));
  // 512 pad rows: the root kernel's bulk copies always move whole tiles (rows past n are masked in the kernel)
  const size_t n_alloc = (size_t)n + 512;
  bins.alloc(n_alloc * ngroups * kSlots); bins_tail.alloc(tw ? n_alloc * tw : 0);
  CUDA_OK(cudaMemsetAsync(bins.p + (size_t)n * ngroups * kSlots, 0, (size_t)512 * ngroups * kSlots, s));
  if (tw) CUDA_OK(cudaMemsetAsync(bins_tail.p + (size_t)n * tw, 0, (size_t)512 * tw, s));
}

void DMatrix::finish_bins() {
  cudaStream_t s = engine_stream();
  gather_stride = ngroups * kSlots;
  bins_gather.release();
  static const bool no_aligned = getenv("B200XGB_NO_ALIGNED_ROWS") != nullptr;
  if (ngroups * kSlots == 96 && !no_aligned) {           // 96 B rows straddle 128 B DRAM lines half of the time: the gathered levels read an aligned copy
    // An 8-wide tail goes into the pad of the line (offset 96): the gathered levels then take it from the line they fetch
    // anyway instead of gathering 8 B from bins_tail by row id.  A 4-wide tail stays out: it travels with the row ids, and a
    // second request per gathered row into the line cost more in the histograms than it saved in the partition (DESIGN §6).
    gather_stride = 128;
    bins_gather.alloc((size_t)n * 128 + 128);
    launch_pad_rows(bins.p, bins_tail.p, tw == 8 ? 8 : 0, n, 96, bins_gather.p, 128, s);
  }
  bins_col.alloc((size_t)std::max(F, 1) * n);
  launch_transpose_bins(bins.p, bins_tail.p, n, F, ngroups, tw, bins_col.p, s);
  Comm::get().sync_stream(s);
  binned = true;
}

void DMatrix::set_cuts(const HostCuts& c) {
  require_raw("XGB200DMatrixSetCuts (re-binning)");
  B200_CHECK((int)c.ptrs.size() == F + 1 && (int)c.mins.size() == F, "SetCuts: cut_ptrs/min_vals do not match the number of features");
  for (int f = 0; f < F; ++f) B200_CHECK(c.ptrs[f + 1] - c.ptrs[f] >= 1 && c.ptrs[f + 1] - c.ptrs[f] <= (has_missing ? 255 : 256), "SetCuts: 1..256 cuts per feature (255 with missing values)");
  cuts = c; binned_max_bin = -1;
  bin_with_cuts();
}

void DMatrix::ensure_binned(int max_bin) {
  if (binned && (binned_max_bin == max_bin || binned_max_bin == -1)) return;
  B200_CHECK(!quantile, "max_bin=" + std::to_string(max_bin) + " differs from the max_bin=" + std::to_string(quantile_max_bin) +
             " this QuantileDMatrix was built with; pass the training max_bin to QuantileDMatrix(max_bin=...)");
  B200_CHECK(max_bin >= 2, "max_bin must be >= 2");
  cudaStream_t s = engine_stream();
  Comm& comm = Comm::get();
  // weights per query group weigh each row of the group in the sketch
  DevBuf<float> row_w;
  const float* w = weights.empty() ? nullptr : d_weights.p;
  if (w && (int64_t)weights.size() != n) {
    B200_CHECK(!group_ptr.empty() && weights.size() == group_ptr.size() - 1, "weights must have one entry per row, or one per query group (" +
               std::to_string(n) + " rows, " + std::to_string(weights.size()) + " weights)");
    std::vector<float> h((size_t)n);
    for (size_t g = 0; g + 1 < group_ptr.size(); ++g) std::fill(h.begin() + group_ptr[g], h.begin() + group_ptr[g + 1], weights[g]);
    row_w.alloc((size_t)n);
    CUDA_OK(cudaMemcpyAsync(row_w.p, h.data(), sizeof(float) * n, cudaMemcpyHostToDevice, s));
    comm.sync_stream(s);
    w = row_w.p;
  }
  if (!comm.distributed()) {
    compute_cuts_device(X.p, n, F, w, max_bin, has_missing, &cuts, s);
  } else {
    // every rank summarises its shard (exact when a feature has <= cap distinct values), the summaries are
    // all-gathered and merged, and every rank derives the same cuts.
    const int cap = kRankSummaryCap;
    int hm = has_missing ? 1 : 0;
    {   // has_missing must agree across ranks (bin code 255 reservation)
      DevBuf<unsigned> flag; flag.alloc(1); unsigned v = (unsigned)hm;
      CUDA_OK(cudaMemcpyAsync(flag.p, &v, 4, cudaMemcpyHostToDevice, s));
      comm.allreduce_max_u32(flag.p, 1, s);
      CUDA_OK(cudaMemcpyAsync(&v, flag.p, 4, cudaMemcpyDeviceToHost, s)); Comm::get().sync_stream(s);
      has_missing = v != 0;
    }
    std::vector<FeatureSummary> local;
    compute_summaries_device(X.p, n, F, w, cap, &local, s);
    const size_t per_feat = (size_t)(cap + 2);
    const size_t rec = per_feat * (sizeof(float) + sizeof(double)) + sizeof(double);   // vals, weights, count
    std::vector<unsigned char> sendbuf((size_t)F * rec, 0);
    for (int f = 0; f < F; ++f) {
      unsigned char* p = sendbuf.data() + (size_t)f * rec;
      double cntd = (double)local[f].vals.size(); memcpy(p, &cntd, 8);
      memcpy(p + 8, local[f].vals.data(), sizeof(float) * local[f].vals.size());
      memcpy(p + 8 + per_feat * sizeof(float), local[f].weights.data(), sizeof(double) * local[f].weights.size());
    }
    const int W = comm.world();
    DevBuf<unsigned char> dsend, drecv; dsend.alloc(sendbuf.size()); drecv.alloc(sendbuf.size() * W);
    CUDA_OK(cudaMemcpyAsync(dsend.p, sendbuf.data(), sendbuf.size(), cudaMemcpyHostToDevice, s));
    comm.allgather_bytes(dsend.p, drecv.p, sendbuf.size(), s);
    std::vector<unsigned char> all(sendbuf.size() * W);
    CUDA_OK(cudaMemcpyAsync(all.data(), drecv.p, all.size(), cudaMemcpyDeviceToHost, s));
    Comm::get().sync_stream(s);
    std::vector<std::vector<FeatureSummary>> per_rank(W, std::vector<FeatureSummary>(F));
    for (int r = 0; r < W; ++r) {
      for (int f = 0; f < F; ++f) {
        const unsigned char* p = all.data() + (size_t)r * sendbuf.size() + (size_t)f * rec;
        double cntd; memcpy(&cntd, p, 8); size_t c = (size_t)cntd;
        FeatureSummary& fs = per_rank[r][f];
        fs.vals.resize(c); fs.weights.resize(c);
        memcpy(fs.vals.data(), p + 8, sizeof(float) * c);
        memcpy(fs.weights.data(), p + 8 + per_feat * sizeof(float), sizeof(double) * c);
      }
    }
    std::vector<FeatureSummary> merged;
    merge_summaries(per_rank, F, &merged);
    cuts_from_summaries(merged, max_bin, has_missing, &cuts);
  }
  binned_max_bin = max_bin;
  bin_with_cuts();
}

// ---------------------------------------------------------------------------------------------
// QuantileDMatrix: binned from batches, no float copy of the whole matrix (DESIGN.md "QuantileDMatrix")
// ---------------------------------------------------------------------------------------------
void ProxyBatch::set_float_info(const std::string& field, const float* v, size_t len) {
  if (field == "label") { labels.assign(v, v + len); label_cols = 1; }
  else if (field == "weight") {
    for (size_t i = 0; i < len; ++i) B200_CHECK(v[i] >= 0 && !std::isnan(v[i]), "Weights must be positive values.");
    weights.assign(v, v + len);
  }
  else if (field == "base_margin") base_margin.assign(v, v + len);
  else if (field == "label_lower_bound") label_lower.assign(v, v + len);
  else if (field == "label_upper_bound") label_upper.assign(v, v + len);
  else throw Error("Unknown float field name: " + field);
}

namespace {
// The proxy's batch as a row-major float matrix on the device with NaN for missing.  A float32 device batch is read in place
// unless it must be copied (copy, or a `missing` other than NaN: the producer's buffer is never written); everything else is
// staged in `scratch`, which grows to the largest batch.  A CSR batch marks missing values by absence and keeps its stored
// values, as DMatrix::from_csr does.  *nmiss: the missing entries.
const float* stage_batch(const ProxyBatch& p, float missing, bool copy, DevBuf<float>& scratch, int64_t* nmiss, cudaStream_t s) {
  B200_CHECK(p.kind != ProxyBatch::kNone, "QuantileDMatrix: the iterator's next() returned true without setting data on the proxy");
  B200_CHECK(p.n >= 0 && p.n < (int64_t)0x7fffffff && p.F >= 0, "QuantileDMatrix: bad batch shape");
  const size_t count = (size_t)p.n * p.F;
  const bool use_missing = !std::isnan(missing) && p.kind != ProxyBatch::kCSR;
  const float* dX = nullptr;
  if (p.kind == ProxyBatch::kDevice) {
    CUDA_OK(cudaDeviceSynchronize());       // the producer (e.g. a torch stream) must be done before we read its buffer
    if (!copy && !use_missing) dX = p.data;
    else { scratch.ensure(std::max<size_t>(count, 1)); if (count) CUDA_OK(cudaMemcpyAsync(scratch.p, p.data, sizeof(float) * count, cudaMemcpyDeviceToDevice, s)); }
  } else if (p.kind == ProxyBatch::kHostDense) {
    scratch.ensure(std::max<size_t>(count, 1));
    const float* src = p.converted.empty() ? p.data : p.converted.data();
    if (count) CUDA_OK(cudaMemcpyAsync(scratch.p, src, sizeof(float) * count, cudaMemcpyHostToDevice, s));
  } else {
    scratch.ensure(std::max<size_t>(count, 1));
    if (count) {
      DevBuf<unsigned long long> d_ptr; DevBuf<unsigned> d_idx; DevBuf<float> d_val;
      d_ptr.alloc((size_t)p.n + 1); d_idx.alloc(std::max<size_t>(p.nelem, 1)); d_val.alloc(std::max<size_t>(p.nelem, 1));
      CUDA_OK(cudaMemcpyAsync(d_ptr.p, p.indptr, sizeof(size_t) * ((size_t)p.n + 1), cudaMemcpyHostToDevice, s));
      if (p.nelem) { CUDA_OK(cudaMemcpyAsync(d_idx.p, p.indices, sizeof(unsigned) * p.nelem, cudaMemcpyHostToDevice, s));
                     CUDA_OK(cudaMemcpyAsync(d_val.p, p.values, sizeof(float) * p.nelem, cudaMemcpyHostToDevice, s)); }
      csr_to_dense_device(d_ptr.p, d_idx.p, d_val.p, p.n, p.F, scratch.p, s);
      Comm::get().sync_stream(s);                 // the staging buffers above die with this scope
    }
  }
  if (!dX) dX = scratch.p;
  DevBuf<unsigned long long> cnt; cnt.alloc(1); cnt.zero(s);
  launch_count_nan(dX, (int64_t)count, missing, use_missing ? 1 : 0, cnt.p, s);
  if (use_missing) launch_replace_missing(scratch.p, (int64_t)count, missing, s);   // dX == scratch.p here
  unsigned long long c = 0;
  CUDA_OK(cudaMemcpyAsync(&c, cnt.p, 8, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  *nmiss = (int64_t)c;
  return dX;
}
}  // namespace

std::unique_ptr<DMatrix> DMatrix::from_batches(ProxyBatch* proxy, const std::function<void()>& reset, const std::function<bool()>& next,
                                               DMatrix* ref, float missing, int max_bin) {
  B200_CHECK(!Comm::get().distributed(), "QuantileDMatrix is not supported with more than one GPU (world_size > 1); build a DMatrix on each worker");
  B200_CHECK(max_bin >= 2, "max_bin must be >= 2");
  if (ref) {
    if (!ref->quantile) ref->ensure_binned(max_bin);
    B200_CHECK(ref->binned, "QuantileDMatrix: ref has no cuts");
  }
  cudaStream_t s = engine_stream();
  auto dm = std::make_unique<DMatrix>();
  dm->quantile = true;
  DevBuf<float> scratch, wbuf;
  std::vector<int64_t> rows;
  std::vector<std::vector<FeatureSummary>> per_batch;
  std::vector<float> labels, weights, base_margin, lower, upper, w0;
  std::vector<int64_t> qid;
  int label_cols = 0;                                 // T of the batches' labels (0: no batch had labels yet)
  int64_t nmiss_total = 0;
  auto summarise = [&](const float* dX, int64_t nr, const std::vector<float>& w) {
    if (!w.empty()) { wbuf.ensure(w.size()); CUDA_OK(cudaMemcpyAsync(wbuf.p, w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice, s)); }
    per_batch.emplace_back();
    compute_summaries_device(dX, nr, dm->F, w.empty() ? nullptr : wbuf.p, kRankSummaryCap, &per_batch.back(), s);
  };
  auto append = [](std::vector<float>& dst, const std::vector<float>& src, int64_t nr, int b, const char* what) {
    B200_CHECK(src.empty() || (int64_t)src.size() == nr || std::string(what) == "base_margin",
               std::string("QuantileDMatrix: batch ") + std::to_string(b) + " has " + std::to_string(src.size()) + " " + what + " for " + std::to_string(nr) + " rows");
    dst.insert(dst.end(), src.begin(), src.end());
  };
  // pass 1: shapes, missing values, meta information, and (without ref) one summary per batch.  Batch 0 is always copied to
  // the scratch buffer: if it is the only batch, it is binned from there with the exact single-rank cuts.
  reset();
  bool more = next();
  int b = 0;
  while (more) {
    const ProxyBatch& p = *proxy;
    if (b == 0) dm->F = p.F;
    B200_CHECK(p.F == dm->F, "QuantileDMatrix: batch " + std::to_string(b) + " has " + std::to_string(p.F) + " columns, the first batch has " + std::to_string(dm->F));
    int64_t nm = 0;
    const float* dX = stage_batch(p, missing, b == 0, scratch, &nm, s);
    nmiss_total += nm; rows.push_back(p.n);
    if (!p.labels.empty()) {
      B200_CHECK(label_cols == 0 || p.label_cols == label_cols, "QuantileDMatrix: batch " + std::to_string(b) + " has a label of " + std::to_string(p.label_cols) +
                 " columns, an earlier batch one of " + std::to_string(label_cols) + "; every batch's label must have the same number of columns");
      label_cols = p.label_cols;
      B200_CHECK((int64_t)p.labels.size() == p.n * p.label_cols, "QuantileDMatrix: batch " + std::to_string(b) + " has " + std::to_string(p.labels.size()) +
                 " labels for " + std::to_string(p.n) + " rows");
      labels.insert(labels.end(), p.labels.begin(), p.labels.end());
    }
    append(weights, p.weights, p.n, b, "weights"); append(base_margin, p.base_margin, p.n, b, "base_margin");
    append(lower, p.label_lower, p.n, b, "label_lower_bound"); append(upper, p.label_upper, p.n, b, "label_upper_bound");
    B200_CHECK(p.qid.empty() || (int64_t)p.qid.size() == p.n, "QuantileDMatrix: batch " + std::to_string(b) + " has " + std::to_string(p.qid.size()) + " qid for " + std::to_string(p.n) + " rows");
    qid.insert(qid.end(), p.qid.begin(), p.qid.end());
    if (b == 0) w0 = p.weights;
    else if (!ref) summarise(dX, p.n, p.weights);          // before next(): the producer may release the batch
    more = next();
    if (b == 0 && more && !ref) summarise(scratch.p, rows[0], w0);
    ++b;
  }
  const int nb = b;
  int64_t n = 0;
  for (int64_t r : rows) n += r;
  B200_CHECK(n < (int64_t)0x7fffffff, "QuantileDMatrix: more than 2^31-1 rows per GPU are not supported");
  dm->n = n;
  dm->has_missing = nmiss_total > 0;
  int F = dm->F;
  if (ref) {
    B200_CHECK(ref->F == F || nb == 0, "QuantileDMatrix: the data has " + std::to_string(F) + " columns, ref has " + std::to_string(ref->F));
    dm->F = F = ref->F;
    dm->cuts = ref->cuts;
    if (dm->has_missing)
      for (int f = 0; f < F; ++f)
        B200_CHECK(ref->cuts.ptrs[f + 1] - ref->cuts.ptrs[f] <= kMissingBin,
                   "QuantileDMatrix: the data has missing values, but the cuts of ref use all 256 bin codes for feature " + std::to_string(f) +
                   " (ref has no missing values), so code 255 cannot mark them; build ref with a missing value, or use a DMatrix");
    dm->binned_max_bin = ref->quantile ? ref->quantile_max_bin : ref->binned_max_bin;
  } else {
    if (nb == 1) {
      if (!w0.empty()) { wbuf.ensure(w0.size()); CUDA_OK(cudaMemcpyAsync(wbuf.p, w0.data(), sizeof(float) * w0.size(), cudaMemcpyHostToDevice, s)); }
      compute_cuts_device(scratch.p, n, F, w0.empty() ? nullptr : wbuf.p, max_bin, dm->has_missing, &dm->cuts, s);
    } else {
      std::vector<FeatureSummary> merged;
      merge_summaries(per_batch, F, &merged);
      cuts_from_summaries(merged, max_bin, dm->has_missing, &dm->cuts);
    }
    dm->binned_max_bin = max_bin;
  }
  per_batch.clear(); wbuf.release();
  dm->quantile_max_bin = dm->binned_max_bin;
  dm->alloc_bins();
  if (nb == 1) {
    if (n) launch_bin(scratch.p, n, F, dm->ngroups, dm->tw, dm->d_cut_ptrs.p, dm->d_cut_vals.p, dm->bins.p, dm->bins_tail.p, s);
  } else if (nb > 1) {
    // pass 2: every batch binned into the final bins at its row offset
    reset();
    int64_t off = 0; int bi = 0;
    while (next()) {
      const ProxyBatch& p = *proxy;
      B200_CHECK(bi < nb, "QuantileDMatrix: the iterator yielded more than the " + std::to_string(nb) + " batches of its first pass");
      B200_CHECK(p.n == rows[bi] && p.F == F, "QuantileDMatrix: batch " + std::to_string(bi) + " is " + std::to_string(p.n) + " x " + std::to_string(p.F) +
                 " in the second pass but was " + std::to_string(rows[bi]) + " x " + std::to_string(F) + " in the first; the iterator must yield the same batches after reset()");
      int64_t nm = 0;
      const float* dX = stage_batch(p, missing, false, scratch, &nm, s);
      if (p.n) launch_bin(dX, p.n, F, dm->ngroups, dm->tw, dm->d_cut_ptrs.p, dm->d_cut_vals.p, dm->bins.p + (size_t)off * dm->ngroups * kSlots,
                          dm->tw ? dm->bins_tail.p + (size_t)off * dm->tw : nullptr, s);
      CUDA_OK(cudaStreamSynchronize(s));      // before next(): the producer may release the batch
      off += p.n; ++bi;
    }
    B200_CHECK(bi == nb, "QuantileDMatrix: the iterator yielded " + std::to_string(bi) + " batches in its second pass and " + std::to_string(nb) + " in its first");
  }
  scratch.release();
  dm->finish_bins();
  B200_CHECK(qid.empty() || weights.empty(), "weights together with query groups are not supported on a QuantileDMatrix");
  auto need_all = [&](const std::vector<float>& v, const char* what) {
    B200_CHECK(v.empty() || (int64_t)v.size() == n, std::string("QuantileDMatrix: ") + what + " must be given for every batch or for none (" +
               std::to_string(v.size()) + " for " + std::to_string(n) + " rows)");
  };
  B200_CHECK(labels.empty() || (int64_t)labels.size() == n * label_cols, "QuantileDMatrix: labels must be given for every batch or for none (" +
             std::to_string(labels.size() / std::max(label_cols, 1)) + " label rows for " + std::to_string(n) + " rows)");
  need_all(weights, "weights"); need_all(lower, "label_lower_bound"); need_all(upper, "label_upper_bound");
  B200_CHECK(qid.empty() || (int64_t)qid.size() == n, "QuantileDMatrix: qid must be given for every batch or for none");
  if (!labels.empty()) dm->set_label_matrix(labels.data(), n, label_cols);
  if (!weights.empty()) dm->set_float_info("weight", weights.data(), weights.size());
  if (!base_margin.empty()) dm->set_float_info("base_margin", base_margin.data(), base_margin.size());
  if (!lower.empty()) dm->set_float_info("label_lower_bound", lower.data(), lower.size());
  if (!upper.empty()) dm->set_float_info("label_upper_bound", upper.data(), upper.size());
  if (!qid.empty()) dm->set_qid(qid.data(), qid.size());
  return dm;
}

// Column sampling (upstream src/common/random.h ColumnSampler: bytree, then bylevel inside it, then bynode inside that; a
// subset keeps max(1, floor(frac * |parent|)) features).  Upstream shuffles with a mt19937; product and oracle share a
// counter-based rule instead: feature f of the parent set is kept iff fewer than `keep` parent features have a smaller
// hash u(stream, f) (ties: lower index first).  Streams: tree 0x1000 + t, level 0x300000 + 64 t + depth, node (eval kernel)
// 0x80000000 + 2^20 t + nid; the gradient subsample (misc.cu) draws from 0x2000 + round.  booster=dart draws its skip from
// kDartSkipStream (index: round), its per-tree drops from kDartTreeStream + round (index: tree) and its one_drop pick from
// kDartOneStream (index: round), all above 2^40 where no other stream reaches.  A forest (num_parallel_tree > 1) draws the
// rows of tree j >= 1 of a round from kForestRowStream + 2^20 round + j (index: row); tree 0 keeps 0x2000 + round.
constexpr uint64_t kDartSkipStream = 0x10000000000ull, kDartOneStream = 0x20000000000ull, kDartTreeStream = 0x30000000000ull;
constexpr uint64_t kForestRowStream = 0x40000000000ull;
// lambdarank_pair_method=mean: draw j of a document of round `round` comes from kRankPairStream + 2^20 round + j (index: row + rank
// offset, as the subsample draw), so lambdarank_num_pair_per_sample is at most 2^20 under mean
constexpr uint64_t kRankPairStream = 0x50000000000ull;
// the stream tree j of boosting round `round` draws its row sample from (uniform and gradient-based sampling alike)
static uint64_t row_stream(int round, int j) { return j == 0 ? 0x2000ull + (uint64_t)round : kForestRowStream + ((uint64_t)round << 20) + (uint64_t)j; }
std::string subset_mask(const std::string& parent, float frac, unsigned seed, uint64_t stream) {
  if (frac >= 1.0f) return parent;
  const int F = (int)parent.size();
  int cnt = 0; for (int f = 0; f < F; ++f) cnt += parent[f] ? 1 : 0;
  const int keep = std::max(1, (int)std::floor(frac * (float)cnt));
  std::vector<float> u(F);
  for (int f = 0; f < F; ++f) u[f] = rng_uniform(seed, stream, (uint64_t)f);
  std::string m((size_t)F, (char)0);
  for (int f = 0; f < F; ++f) {
    if (!parent[f]) continue;
    int rank = 0;
    for (int g = 0; g < F; ++g) if (parent[g] && (u[g] < u[f] || (u[g] == u[f] && g < f))) ++rank;
    m[f] = rank < keep ? 1 : 0;
  }
  return m;
}
std::string colsample_mask(unsigned seed, int tree_index, int F, float frac) {
  return subset_mask(std::string((size_t)F, (char)1), frac, seed, 0x1000 + (uint64_t)tree_index);
}

// ---------------------------------------------------------------------------------------------
// Booster
// ---------------------------------------------------------------------------------------------
Booster::Booster() {}
Booster::~Booster() {
  for (auto& p : pending_) if (p.ready) cudaEventDestroy(p.ready);
}

const std::map<std::string, int>& objective_table() {
  static const std::map<std::string, int> t = {{"reg:squarederror", kSquaredError}, {"reg:linear", kSquaredError}, {"binary:logistic", kBinaryLogistic},
    {"reg:logistic", kRegLogistic}, {"binary:logitraw", kLogitRaw}, {"multi:softprob", kSoftprob}, {"multi:softmax", kSoftmax},
    {"reg:squaredlogerror", kSquaredLogError}, {"reg:pseudohubererror", kPseudoHuber}, {"count:poisson", kPoisson}, {"reg:gamma", kGamma},
    {"reg:tweedie", kTweedie}, {"binary:hinge", kHinge}, {"survival:aft", kAft}, {"survival:cox", kCox}, {"reg:absoluteerror", kAbsoluteError},
    {"reg:quantileerror", kQuantileError}, {"rank:pairwise", kRankPairwise}, {"rank:ndcg", kRankNdcg}, {"rank:map", kRankMap}};
  return t;
}

void Booster::set_param(const std::string& k, const std::string& v) {
  if (k == "eval_metric") { if (std::find(eval_metrics_.begin(), eval_metrics_.end(), v) == eval_metrics_.end()) eval_metrics_.push_back(v); }
  else raw_params_[k] = v;
  configured_ = false;
}

// quantile_alpha: "0.5", the "(0.1,0.5,0.9)" of a Python list or tuple, or the "[0.1, 0.5, 0.9]" of a saved config; at least one
// value, each in [0, 1] [UPSTREAM-RECALL: QuantileLossParam::Validate]
std::vector<float> parse_quantile_alpha(const std::string& v) {
  std::vector<float> out; std::string tok;
  auto flush = [&]() {
    if (tok.empty()) return;
    size_t used = 0; float a = 0.0f;
    try { a = std::stof(tok, &used); } catch (...) { used = 0; }
    B200_CHECK(used > 0 && used == tok.size(), "Invalid value for parameter quantile_alpha: " + v);
    B200_CHECK(a >= 0.0f && a <= 1.0f, "quantile_alpha must be in [0, 1] (got " + tok + ")");
    out.push_back(a); tok.clear();
  };
  for (char ch : v) {
    if (ch == ',' || ch == '(' || ch == ')' || ch == '[' || ch == ']' || std::isspace((unsigned char)ch)) flush();
    else tok.push_back(ch);
  }
  flush();
  B200_CHECK(!out.empty(), "quantile_alpha must not be empty (got \"" + v + "\")");
  return out;
}

void Booster::configure() {
  if (configured_) return;
  auto getf = [&](const char* a, const char* b, float def) { auto it = raw_params_.find(a); if (it == raw_params_.end() && b) it = raw_params_.find(b);
    if (it == raw_params_.end()) return def; try { return std::stof(it->second); } catch (...) { throw Error(std::string("Invalid value for parameter ") + a + ": " + it->second); } };
  auto geti = [&](const char* a, int def) { auto it = raw_params_.find(a); if (it == raw_params_.end()) return def;
    try { return (int)std::stod(it->second); } catch (...) { throw Error(std::string("Invalid value for parameter ") + a + ": " + it->second); } };
  TrainParam p;
  auto ito = raw_params_.find("objective");
  if (ito != raw_params_.end()) objective_name_ = ito->second;
  auto ot = objective_table().find(objective_name_);
  B200_CHECK(ot != objective_table().end(), "Unknown objective function: `" + objective_name_ + "` (supported on the CUDA hist path: reg:squarederror, reg:linear, reg:logistic, reg:squaredlogerror, reg:pseudohubererror, reg:absoluteerror, reg:quantileerror, reg:gamma, reg:tweedie, count:poisson, binary:logistic, binary:logitraw, binary:hinge, multi:softprob, multi:softmax, survival:aft, survival:cox, rank:pairwise, rank:ndcg, rank:map)");
  p.objective = ot->second;
  if (objective_name_ == "reg:linear") objective_name_ = "reg:squarederror";
  p.num_class = (p.objective == kSoftprob || p.objective == kSoftmax) ? geti("num_class", 0) : 1;
  if (p.objective == kSoftprob || p.objective == kSoftmax) B200_CHECK(p.num_class >= 1, "num_class must be set (>= 1) for multi:softprob / multi:softmax");
  p.max_depth = geti("max_depth", 6); p.max_leaves = geti("max_leaves", 0); p.max_bin = geti("max_bin", 256);
  p.eta = getf("eta", "learning_rate", 0.3f); p.lambda = getf("lambda", "reg_lambda", 1.0f); p.alpha = getf("alpha", "reg_alpha", 0.0f);
  p.gamma = getf("gamma", "min_split_loss", 0.0f); p.min_child_weight = getf("min_child_weight", nullptr, 1.0f);
  p.max_delta_step = getf("max_delta_step", nullptr, 0.0f); p.scale_pos_weight = getf("scale_pos_weight", nullptr, 1.0f);
  p.subsample = getf("subsample", nullptr, 1.0f); p.colsample_bytree = getf("colsample_bytree", nullptr, 1.0f);
  p.colsample_bylevel = getf("colsample_bylevel", nullptr, 1.0f); p.colsample_bynode = getf("colsample_bynode", nullptr, 1.0f);
  p.seed = (unsigned)geti("seed", 0);
  if (auto it = raw_params_.find("num_parallel_tree"); it != raw_params_.end()) {
    double v = 0.0; size_t used = 0;
    try { v = std::stod(it->second, &used); } catch (...) { used = 0; }
    while (used > 0 && used < it->second.size() && std::isspace((unsigned char)it->second[used])) ++used;
    B200_CHECK(used > 0 && used == it->second.size() && v == std::floor(v) && v >= 1.0 && v <= (double)(1 << 20), "num_parallel_tree must be an integer in [1, 1048576] (got " + it->second + ")");
    p.num_parallel_tree = (int)v;
  }
  if (p.objective == kQuantileError) {       // quantile_alpha is read (and checked) only under reg:quantileerror
    auto qa = raw_params_.find("quantile_alpha");
    B200_CHECK(qa != raw_params_.end(), "reg:quantileerror needs the parameter quantile_alpha (a value or a list of values in [0, 1])");
    p.quantile_alpha = parse_quantile_alpha(qa->second);
  }
  p.huber_slope = getf("huber_slope", nullptr, 1.0f); p.tweedie_variance_power = getf("tweedie_variance_power", nullptr, 1.5f);
  B200_CHECK(p.huber_slope != 0.0f, "Check failed: slope != 0.0 (huber_slope)");
  B200_CHECK(p.tweedie_variance_power >= 1.0f && p.tweedie_variance_power < 2.0f, "tweedie_variance_power must be in interval [1, 2)");
  if (p.objective == kAft) {      // the AFT parameters are read (and checked) only under survival:aft
    if (auto d = raw_params_.find("aft_loss_distribution"); d != raw_params_.end()) {
      if (d->second == "normal") p.aft_dist = kAftNormal;
      else if (d->second == "logistic") p.aft_dist = kAftLogistic;
      else if (d->second == "extreme") p.aft_dist = kAftExtreme;
      else throw Error("Invalid aft_loss_distribution: " + d->second + " (normal, logistic, extreme)");
    }
    p.aft_sigma = getf("aft_loss_distribution_scale", nullptr, 1.0f);
    B200_CHECK(p.aft_sigma > 0.0f && std::isfinite(p.aft_sigma), "aft_loss_distribution_scale must be a finite number > 0 (got " + std::to_string(p.aft_sigma) + ")");
  }
  if (objective_is_rank(p.objective)) {     // the LambdaRank parameters are read (and checked) only under rank:*
    auto getb = [&](const char* a, int def) {
      auto it = raw_params_.find(a); if (it == raw_params_.end()) return def;
      std::string v = it->second; for (char& ch : v) ch = (char)std::tolower((unsigned char)ch);
      if (v == "1" || v == "true") return 1;
      if (v == "0" || v == "false") return 0;
      throw Error(std::string("Invalid value for parameter ") + a + ": " + it->second + " (true or false)");
    };
    if (auto pm = raw_params_.find("lambdarank_pair_method"); pm != raw_params_.end()) {
      B200_CHECK(pm->second == "topk" || pm->second == "mean", "Invalid value for parameter lambdarank_pair_method: " + pm->second + " (topk, mean)");
      p.rank_mean = pm->second == "mean" ? 1 : 0;
    }
    if (p.rank_mean) p.rank_k = 1;
    if (auto kp = raw_params_.find("lambdarank_num_pair_per_sample"); kp != raw_params_.end()) {
      double v = 0.0; size_t used = 0;
      try { v = std::stod(kp->second, &used); } catch (...) { used = 0; }
      B200_CHECK(used > 0 && used == kp->second.size() && v == std::floor(v) && v >= 1.0 && v <= 2147483647.0,
                 "lambdarank_num_pair_per_sample must be an integer >= 1 (got " + kp->second + ")");
      p.rank_k = (int)v;
    }
    p.rank_exp_gain = getb("ndcg_exp_gain", 1); p.rank_normalization = getb("lambdarank_normalization", 1);
    p.rank_score_normalization = getb("lambdarank_score_normalization", 1);
    p.rank_unbiased = getb("lambdarank_unbiased", 0);
    B200_CHECK(!p.rank_mean || p.rank_k <= (1 << 20), "lambdarank_num_pair_per_sample must be <= 1048576 under lambdarank_pair_method=mean");
    p.rank_bias_norm = getf("lambdarank_bias_norm", nullptr, 2.0f);
    B200_CHECK(p.rank_bias_norm >= 0.0f, "lambdarank_bias_norm must be >= 0");
  }
  // count:poisson: max_delta_step defaults to 0.7 for the objective's hessian AND the tree's leaf clipping (upstream learner.cc sets
  // the shared parameter when the user did not)
  if (p.objective == kPoisson) {
    if (raw_params_.find("max_delta_step") == raw_params_.end()) p.max_delta_step = 0.7f;
    p.poisson_max_delta_step = p.max_delta_step;
    B200_CHECK(p.poisson_max_delta_step >= 0.0f, "max_delta_step must be non-negative for count:poisson");
  }
  B200_CHECK(p.lambda >= 0.0f, "Parameter reg_lambda should be greater equal to 0");
  B200_CHECK(p.subsample > 0.0f && p.subsample <= 1.0f, "Parameter subsample should be in (0, 1]");
  if (auto sm = raw_params_.find("sampling_method"); sm != raw_params_.end()) {
    B200_CHECK(sm->second == "uniform" || sm->second == "gradient_based", "Invalid value for parameter sampling_method: " + sm->second + " (uniform, gradient_based)");
    p.gradient_based = sm->second == "gradient_based" ? 1 : 0;
  }
  auto tm = raw_params_.find("tree_method");
  if (tm != raw_params_.end()) {
    const std::string& t = tm->second;
    B200_CHECK(t == "hist" || t == "auto" || t == "gpu_hist" || t == "approx" || t == "exact",
               "Unknown tree_method: " + t);
    // every method maps onto the device hist builder; exact/approx are accepted for hyperparameter compatibility
  }
  auto bo = raw_params_.find("booster");
  if (bo != raw_params_.end()) B200_CHECK(bo->second == "gbtree" || bo->second == "dart", "Only booster=gbtree and booster=dart are implemented on the CUDA hist path (got " + bo->second + ")");
  dart_ = DartParam{};
  if (bo != raw_params_.end() && bo->second == "dart") {      // the DART parameters are read (and checked) only under booster=dart
    dart_.on = true;
    dart_.rate_drop = getf("rate_drop", nullptr, 0.0f); dart_.skip_drop = getf("skip_drop", nullptr, 0.0f); dart_.one_drop = geti("one_drop", 0);
    B200_CHECK(dart_.rate_drop >= 0.0f && dart_.rate_drop <= 1.0f, "Parameter rate_drop should be in [0, 1]");
    B200_CHECK(dart_.skip_drop >= 0.0f && dart_.skip_drop <= 1.0f, "Parameter skip_drop should be in [0, 1]");
    B200_CHECK(dart_.one_drop == 0 || dart_.one_drop == 1, "Parameter one_drop should be 0 or 1");
    auto st = raw_params_.find("sample_type"), nt = raw_params_.find("normalize_type");
    if (st != raw_params_.end()) {
      B200_CHECK(st->second == "uniform" || st->second == "weighted", "Invalid sample_type: " + st->second + " (uniform, weighted)");
      dart_.sample_type = st->second == "weighted" ? 1 : 0;
    }
    if (nt != raw_params_.end()) {
      B200_CHECK(nt->second == "tree" || nt->second == "forest", "Invalid normalize_type: " + nt->second + " (tree, forest)");
      dart_.normalize_type = nt->second == "forest" ? 1 : 0;
    }
  }
  auto gp = raw_params_.find("grow_policy");
  if (gp != raw_params_.end()) {
    B200_CHECK(gp->second == "depthwise" || gp->second == "lossguide", "Invalid grow_policy: " + gp->second + " (depthwise, lossguide)");
    p.lossguide = gp->second == "lossguide" ? 1 : 0;
  }
  interaction_.clear();
  auto ic = raw_params_.find("interaction_constraints");
  if (ic != raw_params_.end()) {                 // "[[0, 1], [2, 3, 4]]": nested lists of feature indices
    int depth = 0; std::string tok; std::vector<int> cur;
    auto flush = [&]() { if (tok.empty()) return; int v = 0; try { v = std::stoi(tok); } catch (...) { throw Error("Invalid interaction_constraints entry: " + tok); }
      B200_CHECK(v >= 0, "interaction_constraints entries must be feature indices (feature names are not supported)"); cur.push_back(v); tok.clear(); };
    for (char ch : ic->second) {
      if (ch == '[' || ch == '(') { ++depth; }
      else if (ch == ']' || ch == ')') { flush(); if (depth == 2 && !cur.empty()) { interaction_.push_back(cur); cur.clear(); } --depth; }
      else if (ch >= '0' && ch <= '9') tok.push_back(ch);
      else { B200_CHECK(ch == ',' || ch == ' ' || ch == '\t' || ch == '\n' || ch == '"' || ch == '\'', std::string("Invalid character in interaction_constraints: ") + ch); flush(); }
    }
    B200_CHECK(depth == 0, "Unbalanced brackets in interaction_constraints");
  }
  monotone_.clear();
  auto mc = raw_params_.find("monotone_constraints");
  if (mc != raw_params_.end()) {                 // "(1,0,-1)" / "1,0,-1" / "[1, 0, -1]": one entry per feature, missing ones are 0
    std::string tok;
    auto flush = [&]() { if (tok.empty()) return; int v = 0; try { v = std::stoi(tok); } catch (...) { throw Error("Invalid monotone_constraints entry: " + tok); }
      B200_CHECK(v >= -1 && v <= 1, "monotone_constraints entries must be -1, 0 or 1"); monotone_.push_back(v); tok.clear(); };
    for (char ch : mc->second) { if (ch == '-' || ch == '+' || (ch >= '0' && ch <= '9')) tok.push_back(ch); else flush(); }
    flush();
    bool any = false; for (int v : monotone_) any |= v != 0;
    if (!any) monotone_.clear();
  }
  if (p.lossguide) {
    B200_CHECK(p.max_depth >= 0 && p.max_depth <= kMaxDepth, "max_depth must be in [0, 16]");
    B200_CHECK(p.max_leaves > 0 || p.max_depth > 0, "grow_policy=lossguide needs max_leaves > 0 or max_depth > 0");
    B200_CHECK(p.max_leaves <= 4096, "max_leaves above 4096 is not supported by the B200 lossguide builder");
    B200_CHECK(p.colsample_bytree >= 1.0f && p.colsample_bylevel >= 1.0f && p.colsample_bynode >= 1.0f, "column sampling (colsample_*) with grow_policy=lossguide is not implemented by the CUDA hist builder");
  }
  auto bs = raw_params_.find("base_score");
  if (bs != raw_params_.end() && !bs->second.empty()) {
    B200_CHECK(bs->second.find_first_of("[,") == std::string::npos, "base_score: a vector base_score (one value per target) is not supported; give one number (got " +
               bs->second + ")");
    base_score_ = std::stof(bs->second); base_score_set_ = true;
    if (p.objective == kBinaryLogistic || p.objective == kRegLogistic || p.objective == kLogitRaw)
      B200_CHECK(base_score_ > 0.0f && base_score_ < 1.0f, "Check failed: base_score > 0.0f && base_score < 1.0f base_score must be in (0,1) for logistic loss");
  }
  if (auto ms = raw_params_.find("multi_strategy"); ms != raw_params_.end())
    B200_CHECK(ms->second == "one_output_per_tree" || ms->second == "multi_output_tree", "Invalid value for parameter multi_strategy: " + ms->second +
               " (one_output_per_tree, multi_output_tree)");
  p.num_target = num_target_;
  if (!p.lossguide) B200_CHECK(p.max_depth >= 1, "max_depth=" + std::to_string(p.max_depth) + " (no depth limit) needs grow_policy=lossguide with max_leaves; the depth-wise builder takes max_depth in [1, 16]");
  if (p.max_bin > 256) p.max_bin = 256;            // uint8 bin codes (the Python layer warns)
  // process_type=update (upstream GBTree): updater is a list of refresh / prune, "refresh,prune" or the "(refresh,prune)" of a
  // Python list; under process_type=default updater and refresh_leaf are accepted and ignored
  update_mode_ = false; update_ops_.clear(); update_ops_str_.clear(); refresh_leaf_ = 1;
  if (auto pt = raw_params_.find("process_type"); pt != raw_params_.end()) {
    B200_CHECK(pt->second == "default" || pt->second == "update", "Invalid value for parameter process_type: " + pt->second + " (default, update)");
    update_mode_ = pt->second == "update";
  }
  if (update_mode_) {
    auto up = raw_params_.find("updater");
    B200_CHECK(up != raw_params_.end(), "process_type=update needs the parameter updater (refresh and/or prune, e.g. updater=refresh,prune)");
    std::string tok;
    auto flush = [&]() {
      if (tok.empty()) return;
      B200_CHECK(tok == "refresh" || tok == "prune", "Invalid updater under process_type=update: " + tok + " (updater may list refresh and prune only)");
      update_ops_.push_back(tok == "refresh" ? kOpRefresh : kOpPrune);
      update_ops_str_ += (update_ops_str_.empty() ? "" : ",") + tok; tok.clear();
    };
    for (char ch : up->second) {
      if (ch == ',' || ch == '(' || ch == ')' || ch == '[' || ch == ']' || ch == '\'' || ch == '"' || std::isspace((unsigned char)ch)) flush();
      else tok.push_back(ch);
    }
    flush();
    B200_CHECK(!update_ops_.empty(), "process_type=update needs the parameter updater (refresh and/or prune, e.g. updater=refresh,prune)");
    B200_CHECK(update_ops_.size() <= (size_t)kMaxRefreshOps, "updater lists more than " + std::to_string(kMaxRefreshOps) + " updaters");
    refresh_leaf_ = geti("refresh_leaf", 1);
    B200_CHECK(refresh_leaf_ == 0 || refresh_leaf_ == 1, "Parameter refresh_leaf should be 0 or 1");
  }
  param_ = p;
  configured_ = true;
}

float Booster::base_margin() const {
  if (objective_is_logistic(param_.objective)) return -std::log(1.0f / base_score_ - 1.0f);
  if (objective_is_log_link(param_.objective) || objective_is_survival(param_.objective)) return std::log(base_score_);   // ProbToMargin of the log-link objectives
  return base_score_;
}

static float objective_aux(const TrainParam& p) {
  switch (p.objective) { case kPseudoHuber: return p.huber_slope; case kTweedie: return p.tweedie_variance_power; case kPoisson: return p.poisson_max_delta_step; default: return 0.0f; }
}

// One Newton stump at margin 0, then PredTransform (upstream src/objective/init_estimation.cc, src/tree/fit_stump.cc)
void Booster::estimate_base_score(DMatrix* dtrain) {
  if (base_score_set_ || base_score_estimated_ || !trees_.empty()) { base_score_estimated_ = true; return; }
  base_score_estimated_ = true;
  if (param_.objective == kSoftprob || param_.objective == kSoftmax) { base_score_ = 0.5f; return; }
  // 3.0.x fits the intercept for the RegLossObj family only; the log-link objectives and binary:hinge keep the 0.5 default
  // [UPSTREAM-RECALL: src/objective/init_estimation.cc; later releases changed the GLM objectives]
  if (objective_is_log_link(param_.objective) || param_.objective == kHinge || objective_is_survival(param_.objective) || objective_is_rank(param_.objective)) { base_score_ = 0.5f; return; }
  cudaStream_t s = engine_stream();
  TreeBuilder& b = *builder_;
  const int T = param_.num_target;
  if (param_.objective == kAbsoluteError) {
    // the median of the labels over every rank's rows, weighted when there are weights (on the fixed-point grid of the
    // weights, adaptive.h); upstream averages each worker's median [UPSTREAM-RECALL: MeanAbsoluteError::InitEstimation]
    // sizing the refresh's buffers first (and dropping any captured tree if they move) leaves none for the select to move.
    // Multi-target: the mean of the T columns' medians, in double, in target order (DESIGN.md "Multi-target regression")
    b.ensure_adaptive(param_.num_outputs());
    DevBuf<float> col; if (T > 1) col.alloc((size_t)std::max<int64_t>(dtrain->n, 1));
    double sum = 0.0;
    for (int j = 0; j < T; ++j) {
      if (T > 1) launch_label_column(dtrain->d_labels.p, dtrain->n, T, j, col.p, s);
      float med = 0.0f;
      segmented_quantile(T > 1 ? col.p : dtrain->d_labels.p, nullptr, dtrain->weights.empty() ? nullptr : dtrain->d_weights.p, dtrain->n, b.global_n, 1, 0.5,
                         &med, &b.adapt, s);
      sum += std::isnan(med) ? 0.0 : (double)med;
    }
    base_score_ = (float)(sum / (double)T);
    return;
  }
  if (param_.objective == kQuantileError) {
    // the mean of the labels' alpha_j-quantiles over every rank's rows (weighted when there are weights), times sw / (sw + 1e-6)
    // with sw the weight sum (the row count without weights), in double [UPSTREAM-RECALL: QuantileRegression::InitEstimation
    // averages the per-alpha quantiles into one scalar; upstream takes each worker's own quantiles]
    b.ensure_adaptive(param_.num_outputs());
    double meanq = 0.0;
    for (float alpha : param_.quantile_alpha) {
      float q = 0.0f;
      segmented_quantile(dtrain->d_labels.p, nullptr, dtrain->weights.empty() ? nullptr : dtrain->d_weights.p, dtrain->n, b.global_n, 1, (double)alpha,
                         &q, &b.adapt, s);
      meanq += std::isnan(q) ? 0.0 : (double)q;
    }
    meanq /= (double)param_.quantile_alpha.size();
    double sw = 0.0;
    if (dtrain->weights.empty()) sw = (double)b.global_n;
    else {
      for (float w : dtrain->weights) sw += (double)w;
      if (Comm::get().distributed()) {
        dsum_.ensure(4);
        CUDA_OK(cudaMemcpyAsync(dsum_.p, &sw, sizeof sw, cudaMemcpyHostToDevice, s));
        Comm::get().allreduce_sum_f64(dsum_.p, 1, s);
        CUDA_OK(cudaMemcpyAsync(&sw, dsum_.p, sizeof sw, cudaMemcpyDeviceToHost, s));
        Comm::get().sync_stream(s);
      }
    }
    base_score_ = (float)(meanq * sw / (sw + 1e-6));
    return;
  }
  // Multi-target: each target's stump as the single-target one, then their mean in margin space, in double, in target order
  // [UPSTREAM-RECALL: FitIntercept::InitEstimation fits the stump of every target, takes their mean, then PredTransform]
  const size_t nsum = std::max<size_t>(4, 2 * (size_t)T);
  dsum_.ensure(nsum);
  CUDA_OK(cudaMemsetAsync(dsum_.p, 0, nsum * sizeof(double), s));
  if (T == 1) {
    GradArgs ga{}; ga.margin = nullptr; ga.label = dtrain->d_labels.p; ga.weight = dtrain->weights.empty() ? nullptr : dtrain->d_weights.p;
    ga.gpair = b.gpair.p; ga.gp_stride = b.gp_stride; ga.absmax = nullptr; ga.err = b.err.p; ga.n = dtrain->n; ga.row_offset = 0; ga.K = 1; ga.objective = param_.objective;
    ga.scale_pos_weight = param_.scale_pos_weight; ga.subsample = 1.0f; ga.seed = 0; ga.iter = 0; ga.aux = objective_aux(param_);
    launch_gradient(ga, s);
  } else {
    MultiGradArgs ma{}; ma.margin = nullptr; ma.label = dtrain->d_labels.p; ma.weight = dtrain->weights.empty() ? nullptr : dtrain->d_weights.p;
    ma.gpair = b.gpair.p; ma.resid = nullptr; ma.absmax = nullptr; ma.err = b.err.p; ma.n = dtrain->n; ma.row_offset = 0; ma.gp_stride = b.gp_stride;
    ma.T = T; ma.objective = param_.objective; ma.per_target = 0; ma.scale_pos_weight = param_.scale_pos_weight; ma.subsample = 1.0f;
    ma.aux = objective_aux(param_); ma.seed = 0; ma.iter = 0;
    launch_multi_target_gradient(ma, s);
  }
  for (int j = 0; j < T; ++j) launch_sum_gpair(b.gpair.p + (size_t)j * b.gp_stride, dtrain->n, dsum_.p + 2 * j, s);
  Comm::get().allreduce_sum_f64(dsum_.p, 2 * (size_t)T, s);
  std::vector<double> h(2 * (size_t)T);
  CUDA_OK(cudaMemcpyAsync(h.data(), dsum_.p, h.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  double wsum = 0.0;
  for (int j = 0; j < T; ++j) wsum += (double)(h[2 * j + 1] <= 0.0 ? 0.0f : (float)(-h[2 * j] / h[2 * j + 1]));
  float w = (float)(wsum / (double)T);
  // binary:logitraw keeps base_score in probability space like the other logistic objectives (the estimated stump weight
  // w is a margin; storing it raw and taking its logit again gives NaN whenever w <= 0, i.e. whenever mean(y) < 0.5)
  if (param_.objective == kBinaryLogistic || param_.objective == kRegLogistic || param_.objective == kLogitRaw) {
    float x = std::min(-w, 88.7f); base_score_ = 1.0f / (std::exp(x) + 1.0f + 1e-16f);
  } else base_score_ = w;
}

void Booster::append_device_tree(int class_id, size_t device_offset, int max_nodes, PendingTree pt, float weight) {
  trees_.emplace_back(); tree_info_.push_back(class_id); pending_.push_back(pt); on_device_.push_back(1); weight_drop_.push_back(weight);
  h_tree_offset.resize(trees_.size() + 1);
  h_tree_offset[trees_.size() - 1] = (int64_t)device_offset;
  h_tree_offset[trees_.size()] = (int64_t)device_offset + max_nodes;
  ++model_version_;
}

void Booster::sync_model() {
  for (size_t t = 0; t < pending_.size(); ++t) {
    PendingTree& p = pending_[t];
    if (!p.staging) continue;
    CUDA_OK(cudaEventSynchronize(p.ready));
    const TreeBlock b = tree_block_layout(p.staging, p.cap_nodes);
    const int nn = *b.n_nodes; const TreeArrays& a = b.t; HostTree& h = trees_[t];
    h.left.assign(a.left, a.left + nn); h.right.assign(a.right, a.right + nn); h.parent.assign(a.parent, a.parent + nn);
    h.split_index.assign(a.split_index, a.split_index + nn); h.split_bin.assign(a.split_bin, a.split_bin + nn); h.split_cond.assign(a.split_cond, a.split_cond + nn);
    h.base_weight.assign(a.base_weight, a.base_weight + nn); h.loss_chg.assign(a.loss_chg, a.loss_chg + nn); h.sum_hess.assign(a.sum_hess, a.sum_hess + nn);
    h.default_left.assign(a.default_left, a.default_left + nn);
    builder_->free_events.push_back(p.ready); p.ready = nullptr; p.staging = nullptr;
  }
  builder_->pinned.reset();
}

void Booster::reserve_nodes(size_t count, size_t slack) {
  if (d_nodes_used + count <= d_nodes.n) return;
  cudaStream_t s = engine_stream();
  DevBuf<DevNode> nb; nb.alloc(std::max<size_t>(d_nodes.n * 2, d_nodes_used + count + slack));
  if (d_nodes_used) CUDA_OK(cudaMemcpyAsync(nb.p, d_nodes.p, sizeof(DevNode) * d_nodes_used, cudaMemcpyDeviceToDevice, s));
  Comm::get().sync_stream(s);
  std::swap(nb.p, d_nodes.p); std::swap(nb.n, d_nodes.n);
}

// make sure every tree is present in the device model (trees loaded from a file are uploaded here)
void Booster::upload_model() {
  cudaStream_t s = engine_stream();
  const int nt = (int)trees_.size();
  if ((int)h_tree_offset.size() != nt + 1) h_tree_offset.resize(nt + 1, 0);
  pending_.resize(nt); on_device_.resize(nt, 0);
  for (int t = 0; t < nt; ++t) {
    if (on_device_[t]) continue;
    const HostTree& h = trees_[t];
    const int nn = h.num_nodes();
    std::vector<DevNode> nodes(nn);
    for (int i = 0; i < nn; ++i) { nodes[i].cond = h.split_cond[i]; nodes[i].left = h.left[i]; nodes[i].right = h.right[i]; nodes[i].fidx_dl = (unsigned)h.split_index[i] | ((unsigned)h.default_left[i] << 31);
      if (h.left[i] >= 0 && h.right[i] != h.left[i] + 1) children_adjacent_ = false; }     // foreign model: the tiled predictor assumes sibling pairs
    reserve_nodes(nn, 4096);
    CUDA_OK(cudaMemcpyAsync(d_nodes.p + d_nodes_used, nodes.data(), sizeof(DevNode) * nn, cudaMemcpyHostToDevice, s));
    Comm::get().sync_stream(s);
    h_tree_offset[t] = (int64_t)d_nodes_used; h_tree_offset[t + 1] = (int64_t)d_nodes_used + nn;
    d_nodes_used += nn; on_device_[t] = 1; d_trees_uploaded = 0;
  }
  if (d_trees_uploaded != nt || d_tree_offset.n < (size_t)nt + 1) {
    d_tree_offset.ensure(std::max<size_t>(nt + 1, 64)); d_tree_info.ensure(std::max<size_t>(nt, 64));
    // offsets are per-tree starts (trees trained on the device have fixed-capacity slots, so starts are not cumulative)
    CUDA_OK(cudaMemcpyAsync(d_tree_offset.p, h_tree_offset.data(), sizeof(int64_t) * (nt + 1), cudaMemcpyHostToDevice, s));
    if (nt) CUDA_OK(cudaMemcpyAsync(d_tree_info.p, tree_info_.data(), sizeof(int) * nt, cudaMemcpyHostToDevice, s));
    Comm::get().sync_stream(s);
    d_trees_uploaded = nt;
  }
}

PredCache& Booster::cache_for(DMatrix* dm) {
  PredCache& c = caches_[dm->uid];
  const int K = param_.num_outputs();
  if (c.n != dm->n || c.margin.n != (size_t)dm->n * K) {
    c.n = dm->n; c.margin.alloc((size_t)dm->n * K); c.trees_applied = -1;
  }
  return c;
}

void Booster::bring_cache_up_to_date(DMatrix* dm, PredCache& c) {
  cudaStream_t s = engine_stream();
  const int K = param_.num_outputs();
  const int nt = (int)trees_.size();
  if (c.trees_applied < 0) {
    if (!dm->base_margin.empty()) {
      B200_CHECK(dm->base_margin.size() == (size_t)dm->n * K, "base_margin size does not match rows x groups");
      CUDA_OK(cudaMemcpyAsync(c.margin.p, dm->d_base_margin.p, sizeof(float) * dm->n * K, cudaMemcpyDeviceToDevice, s));
    } else launch_fill(c.margin.p, dm->n * K, base_margin(), s);
    c.trees_applied = 0; c.weights.clear();
  }
  if (dart_.on) {
    // booster=dart: first fl(w_now - w_applied) * leaf for the trees whose weight changed since, then the new trees with their
    // weights, in one pass of the weighted tree-list kernel
    dm->require_raw("booster=dart");
    std::vector<int> ids; std::vector<float> coef;
    for (int t = 0; t < c.trees_applied; ++t)
      if (c.weights[t] != weight_drop_[t]) { ids.push_back(t); coef.push_back(weight_drop_[t] - c.weights[t]); }
    for (int t = c.trees_applied; t < nt; ++t) { ids.push_back(t); coef.push_back(weight_drop_[t]); }
    if (!ids.empty()) dart_margin(dm, ids, coef, {}, c.margin.p, nullptr);
  } else if (c.trees_applied < nt) {
    upload_model();
    PredictArgs pa = predict_args(dm, c.trees_applied, nt);
    pa.margin = c.margin.p;
    run_predict(dm, pa, s);
  }
  c.trees_applied = nt;
  c.weights.assign(weight_drop_.begin(), weight_drop_.begin() + nt);
}

// ---------------------------------------------------------------------------------------------
// booster=dart (upstream src/gbm/gbtree.cc Dart: DropTrees, NormalizeTrees), with this project's counter-based draws
// ---------------------------------------------------------------------------------------------
// The drop set D of boosting round `round` over the trees so far (T of them, every class), drawn from the streams listed at
// subset_mask: skip_drop decides first, then one draw per tree, then the one_drop pick when D came out empty.
std::vector<int> Booster::dart_drop_set(int round) const {
  std::vector<int> D;
  const int T = (int)weight_drop_.size();
  const unsigned seed = param_.seed;
  if (T == 0) return D;
  if (dart_.skip_drop > 0.0f && rng_uniform(seed, kDartSkipStream, (uint64_t)round) < dart_.skip_drop) return D;
  const uint64_t tree_stream = kDartTreeStream + (uint64_t)round;
  float sum_w = 0.0f;
  for (float w : weight_drop_) sum_w += w;
  for (int i = 0; i < T; ++i) {
    const float u = rng_uniform(seed, tree_stream, (uint64_t)i);
    const float thr = dart_.sample_type == 1 ? dart_.rate_drop * (float)T * weight_drop_[i] / sum_w : dart_.rate_drop;
    if (u < thr) D.push_back(i);
  }
  if (dart_.one_drop && D.empty()) {
    const double u = (double)rng_uniform(seed, kDartOneStream, (uint64_t)round);
    int pick = std::min(T - 1, (int)(u * (double)T));          // uniform
    if (dart_.sample_type == 1) {                                 // in proportion to the weights: first tree whose prefix sum exceeds u * sum
      double tot = 0.0; for (float w : weight_drop_) tot += (double)w;
      const double target = u * tot; double acc = 0.0; pick = T - 1;
      for (int i = 0; i < T; ++i) { acc += (double)weight_drop_[i]; if (acc > target) { pick = i; break; } }
    }
    D.push_back(pick);
  }
  return D;
}

// Draws D, updates the weights of the dropped trees and, in one pass over the rows, the training cache with them; returns
// the margin the round's gradients read (the cache itself when nothing is dropped).  The new trees' weight goes to the builder.
float* Booster::dart_begin_round(DMatrix* dtrain, PredCache& c, int round) {
  const std::vector<int> D = dart_drop_set(round);
  const int K = param_.num_outputs();
  const float lr = (float)((double)param_.eta / (double)K);
  float factor = 1.0f; dart_new_weight_ = 1.0f;
  if (!D.empty()) {
    if (dart_.normalize_type == 1) { factor = (float)(1.0 / (1.0 + (double)lr)); dart_new_weight_ = factor; }
    else { const float denom = (float)D.size() + lr; factor = (float)((double)D.size() / (double)denom); dart_new_weight_ = (float)(1.0 / (double)denom); }
  }
  builder_->set_leaf_scale(dart_new_weight_);
  if (D.empty()) return c.margin.p;
  std::vector<float> coef_full, coef_drop;
  for (int j : D) {
    const float w = weight_drop_[j], w2 = w * factor;
    coef_drop.push_back(w); coef_full.push_back(w2 - w);
    weight_drop_[j] = w2; c.weights[j] = w2;
  }
  dart_drop_margin_.ensure((size_t)dtrain->n * K);
  dart_margin(dtrain, D, coef_full, coef_drop, c.margin.p, dart_drop_margin_.p);
  return dart_drop_margin_.p;
}

void Booster::dart_margin(DMatrix* dm, const std::vector<int>& ids, const std::vector<float>& coef_full, const std::vector<float>& coef_drop,
                          float* m_full, float* m_drop) {
  cudaStream_t s = engine_stream();
  upload_model();
  const size_t m = ids.size();
  dart_ids_.ensure(m); dart_coef_.ensure(2 * m);
  CUDA_OK(cudaMemcpyAsync(dart_ids_.p, ids.data(), sizeof(int) * m, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dart_coef_.p, coef_full.data(), sizeof(float) * m, cudaMemcpyHostToDevice, s));
  if (m_drop) CUDA_OK(cudaMemcpyAsync(dart_coef_.p + m, coef_drop.data(), sizeof(float) * m, cudaMemcpyHostToDevice, s));
  DartArgs a{}; a.X = dm->X.p; a.n = dm->n; a.F = dm->F; a.nodes = d_nodes.p; a.tree_offset = d_tree_offset.p; a.tree_info = d_tree_info.p;
  a.trees = dart_ids_.p; a.ntrees = (int)m; a.K = param_.num_outputs(); a.coef_full = dart_coef_.p; a.coef_drop = dart_coef_.p + m;
  a.m_full = m_full; a.m_drop = m_drop;
  launch_dart_margin(a, s);
  Comm::get().sync_stream(s);            // the host vectors and the list buffers are reused by the next call
}

static void check_labels(const DMatrix* dm) {
  B200_CHECK(dm->labels.size() == (size_t)dm->n * dm->label_cols, "Check failed: preds.size() == info.labels_.size() (" + std::to_string(dm->n) + " vs. " +
             std::to_string(dm->labels.size()) + ") : labels are not correctly provided");
}
// survival:aft reads the interval bounds instead of the label
static void check_aft_bounds(const DMatrix* dm) {
  B200_CHECK(dm->label_lower.size() == (size_t)dm->n && dm->label_upper.size() == (size_t)dm->n,
             "survival:aft needs label_lower_bound and label_upper_bound with one entry per row (" + std::to_string(dm->n) + " rows, " +
             std::to_string(dm->label_lower.size()) + " lower and " + std::to_string(dm->label_upper.size()) + " upper bounds)");
}
// every objective and metric but the ranking ones reads one weight per row
static void check_row_weights(const DMatrix* dm) {
  B200_CHECK(dm->weights.empty() || (int64_t)dm->weights.size() == dm->n, "weights must have one entry per row (" + std::to_string(dm->n) + " rows, " +
             std::to_string(dm->weights.size()) + " weights); one weight per query group is read by the rank:* objectives and the ndcg / map metrics only");
}
static void check_train_width(const DMatrix* dm) {
  B200_CHECK(dm->F <= kMaxTrainFeatures, "the CUDA hist builder trains on at most " + std::to_string(kMaxTrainFeatures) + " features (the data has " +
             std::to_string(dm->F) + ")");
}

void Booster::check_targets(const DMatrix* dm, bool training) {
  configure();
  const int T = dm->label_cols;
  if (T > 1) {
    // [UPSTREAM-RECALL: ObjFunction::Targets defaults to "multioutput is not supported by the current objective function"]
    B200_CHECK(objective_is_multi_target(param_.objective), "multi-target: the label has " + std::to_string(T) + " columns, but objective " + objective_name_ +
               " does not support a label with more than one column (multioutput is not supported by the current objective function); the multi-target "
               "objectives are reg:squarederror, reg:squaredlogerror, reg:pseudohubererror, reg:logistic, binary:logistic, binary:logitraw and reg:absoluteerror");
    auto ms = raw_params_.find("multi_strategy");
    B200_CHECK(ms == raw_params_.end() || ms->second != "multi_output_tree", "multi-target: multi_strategy=multi_output_tree (one tree with a vector leaf for all "
               "targets) is not implemented on the CUDA hist path; use multi_strategy=one_output_per_tree");
    B200_CHECK(!update_mode_, "multi-target: process_type=update is not implemented for a label with more than one column");
  }
  if (training && T != num_target_ && layers() == 0 && !update_mode_) { num_target_ = T; configured_ = false; configure(); }
  B200_CHECK(T == num_target_, "multi-target: the label has " + std::to_string(T) + " column(s) but the model has num_target = " + std::to_string(num_target_));
}

// label-range errors must surface from update() (the container maps them to UserError, train.py:461-467)
void Booster::check_label_ranges(const DMatrix* dtrain) {
  const int K = param_.num_class;
  if (!labels_checked_) {
    const std::vector<float>& y = dtrain->labels;
    if (param_.objective == kBinaryLogistic || param_.objective == kRegLogistic || param_.objective == kLogitRaw)
      for (float v : y) B200_CHECK(v >= 0.0f && v <= 1.0f, "Check failed: label must be in [0,1] for logistic regression");
    if (param_.objective == kSoftprob || param_.objective == kSoftmax)
      for (float v : y) B200_CHECK(v >= 0.0f && (int)v < K, "SoftmaxMultiClassObj: label must be in [0, num_class).");
    if (param_.objective == kSquaredLogError) for (float v : y) B200_CHECK(v > -1.0f, "Check failed: label must be greater than -1 for rmsle so that log(label + 1) can be valid.");
    if (param_.objective == kPoisson) for (float v : y) B200_CHECK(v >= 0.0f, "PoissonRegression: label must be nonnegative");
    if (param_.objective == kGamma) for (float v : y) B200_CHECK(v > 0.0f, "GammaRegression: label must be positive.");
    if (param_.objective == kTweedie) for (float v : y) B200_CHECK(v >= 0.0f, "TweedieRegression: label must be nonnegative");
    if (param_.objective == kAbsoluteError) for (float v : y) B200_CHECK(!std::isnan(v), "reg:absoluteerror: label must not be NaN");
    if (param_.objective == kQuantileError) for (float v : y) B200_CHECK(!std::isnan(v), "reg:quantileerror: label must not be NaN");
    if (objective_is_rank(param_.objective)) for (float v : y) B200_CHECK(!std::isnan(v), objective_name_ + ": label must not be NaN");
    if (param_.objective == kRankNdcg) for (float v : y) {
      B200_CHECK(v >= 0.0f, "rank:ndcg: label must be >= 0 (got " + std::to_string(v) + ")");
      B200_CHECK(!param_.rank_exp_gain || v <= 31.0f, "rank:ndcg: label must be <= 31 with ndcg_exp_gain=true (got " + std::to_string(v) + "); set ndcg_exp_gain=false for larger relevance degrees");
    }
    if (param_.objective == kRankMap) for (float v : y) B200_CHECK(v == 0.0f || v == 1.0f, "rank:map: label must be 0 or 1 (got " + std::to_string(v) + ")");
    if (param_.objective == kAft)
      for (int64_t i = 0; i < dtrain->n; ++i) {
        const float lo = dtrain->label_lower[i], hi = dtrain->label_upper[i];
        B200_CHECK(lo >= 0.0f, "survival:aft: label_lower_bound must be >= 0 (row " + std::to_string(i) + ": " + std::to_string(lo) + ")");
        B200_CHECK(hi >= lo, "survival:aft: label_upper_bound must be >= label_lower_bound (row " + std::to_string(i) + ": " + std::to_string(lo) + " > " + std::to_string(hi) + ")");
      }
    labels_checked_ = true;
  }
}

void Booster::update_one_iter(int iter, DMatrix* dtrain) {
  configure();
  (void)iter;
  cudaStream_t s = engine_stream();
  if (param_.objective == kAft) check_aft_bounds(dtrain); else { check_targets(dtrain, true); check_labels(dtrain); }
  B200_CHECK(param_.objective != kCox || !Comm::get().distributed(), "survival:cox is not supported with more than one GPU (world_size > 1): its risk sets span the rows of every rank");
  if (num_feature_ == 0) num_feature_ = dtrain->F;
  B200_CHECK(num_feature_ == dtrain->F, "Check failed: learner_model_param_.num_feature == p_fmat->Info().num_col_ (" + std::to_string(num_feature_) +
             " vs. " + std::to_string(dtrain->F) + ") : Number of columns does not match number of features in booster.");
  B200_CHECK(dtrain->n > 0 || Comm::get().distributed(), "Empty dataset at worker: 0");
  if (objective_is_rank(param_.objective)) rank_groups(dtrain, objective_name_.c_str());
  else check_row_weights(dtrain);
  if (update_mode_) { dtrain->require_raw("process_type=update"); refresh_one_iter(dtrain); return; }    // reads no bins: no binning, no width limit
  if (dart_.on) dtrain->require_raw("booster=dart");
  check_train_width(dtrain);
  dtrain->ensure_binned(param_.max_bin);
  const int K = param_.num_outputs();
  TreeBuilder& b = builder_for(dtrain);
  check_label_ranges(dtrain);
  estimate_base_score(dtrain);
  PredCache& cache = cache_for(dtrain);
  bring_cache_up_to_date(dtrain, cache);

  const int round = layers();
  const int P = param_.num_parallel_tree;
  // a forest with row sampling draws one row sample per tree: the gradients of every row go to a round buffer first, and each
  // tree's masked copy (and its scales) is made before the tree is grown.  Otherwise every tree of the round shares them.
  const bool per_tree_sample = P > 1 && param_.subsample < 1.0f;
  // sampling_method=gradient_based: the objective writes every row's pairs, each class's threshold is taken once per round on
  // them (the P trees of a forest share it and differ in their draws), and each tree keeps its rows by it
  const bool gbs = gradient_based_sampling();
  // dart forests (a dart model written elsewhere with num_parallel_tree > 1) load and predict, but do not train on
  B200_CHECK(!dart_.on || P == 1, "booster=dart with num_parallel_tree > 1 is not implemented on the CUDA hist path");
  if (!per_tree_sample) forest_gpair_.release();
  // booster=dart: the gradients see the margin without the dropped trees; the cache already holds their new weights
  const float* grad_margin = dart_.on ? dart_begin_round(dtrain, cache, round) : cache.margin.p;
  // ---- gradients + fixed-point scales
  const bool dense_g = constant_hessian(*dtrain);
  // constant-hessian growth needs subsample >= 1, so a per-tree row sample (which copies (g,h) pairs) never sees dense g
  B200_CHECK(!(dense_g && per_tree_sample), "per-tree row sampling of a constant-hessian round");
  // likewise constant-hessian growth never meets a gradient-based sample, whose kept rows have h / p != 1
  B200_CHECK(!(dense_g && gbs), "gradient-based sampling of a constant-hessian round");
  CUDA_OK(cudaMemsetAsync(b.gs.absmax, 0, 8, s));
  // reg:quantileerror and multi-target models without a per-tree or gradient-based sample: each target's trees grow on the grid
  // of its own gradients (upstream quantises each tree's gradients by themselves), so a target's trees do not depend on the
  // other targets
  const bool per_target_grid = (param_.objective == kQuantileError || param_.num_target > 1) && !per_tree_sample && !gbs;
  // reg:absoluteerror / reg:quantileerror: the round's residuals of every output, read by the leaf refresh of every tree of the round
  float* resid = objective_is_adaptive(param_.objective) ? b.ensure_adaptive(K) : nullptr;
  if (per_tree_sample) {
    forest_gpair_.ensure((size_t)b.gp_stride * K);
    launch_objective(dtrain, grad_margin, round, forest_gpair_.p, b.gp_stride, nullptr, 1.0f, false, resid);
    if (gbs) gradient_based_threshold(forest_gpair_.p, b.gp_stride, dtrain->n, K, param_.subsample, &gbs_, s);
  } else if (gbs) {          // one tree per class: sampled in place
    launch_objective(dtrain, grad_margin, round, b.gpair.p, b.gp_stride, nullptr, 1.0f, false, resid);
    gradient_based_threshold(b.gpair.p, b.gp_stride, dtrain->n, K, param_.subsample, &gbs_, s);
    gradient_based_sample(b.gpair.p, b.gpair.p, b.gp_stride, dtrain->n, round, 0, b.gs.absmax);
  } else if (per_target_grid) {
    target_absmax_.ensure(2 * (size_t)K);
    CUDA_OK(cudaMemsetAsync(target_absmax_.p, 0, 2 * sizeof(unsigned) * K, s));
    launch_objective(dtrain, grad_margin, round, b.gpair.p, b.gp_stride, target_absmax_.p, param_.subsample, dense_g, resid, true);
  } else launch_objective(dtrain, grad_margin, round, b.gpair.p, b.gp_stride, b.gs.absmax, param_.subsample, dense_g, resid);
  // weighted adaptive objectives under gradient-based sampling: the refresh weighs its rows by their instance weight (h is w / p)
  if (gbs && resid && !dtrain->weights.empty()) weight_grid(dtrain->d_weights.p, dtrain->n, b.global_n, &b.adapt, s);
  if (per_target_grid) Comm::get().allreduce_max_u32(target_absmax_.p, 2 * (size_t)K, s);
  else if (!per_tree_sample) {
    Comm::get().allreduce_max_u32(b.gs.absmax, 2, s);
    launch_scales(b.gs, grad_bits_for(b.global_n), s);
  }

  // K * P trees, class-major: tree j of class k is tree k * P + j of the layer
  for (int k = 0; k < K; ++k)
    for (int j = 0; j < P; ++j) {
      if (per_tree_sample) {     // tree j's rows (shared by the K classes): j = 0 draws the stream a single tree draws
        CUDA_OK(cudaMemsetAsync(b.gs.absmax, 0, 8, s));
        if (gbs) gradient_based_sample(forest_gpair_.p, b.gpair.p, b.gp_stride, dtrain->n, round, j, b.gs.absmax);
        else {
          SampleArgs sa{}; sa.src = forest_gpair_.p; sa.dst = b.gpair.p; sa.absmax = b.gs.absmax; sa.gp_stride = b.gp_stride; sa.n = dtrain->n;
          sa.row_offset = (int64_t)Comm::get().rank() << 40; sa.K = K; sa.subsample = param_.subsample; sa.seed = param_.seed;
          sa.stream = row_stream(round, j);
          launch_sample_gpair(sa, s);
        }
        Comm::get().allreduce_max_u32(b.gs.absmax, 2, s);
        launch_scales(b.gs, grad_bits_for(b.global_n), s);
      } else if (per_target_grid && j == 0) {
        CUDA_OK(cudaMemcpyAsync(b.gs.absmax, target_absmax_.p + 2 * k, 2 * sizeof(unsigned), cudaMemcpyDeviceToDevice, s));
        launch_scales(b.gs, grad_bits_for(b.global_n), s);
      }
      grow_one_tree(dtrain, cache, k, iteration_indptr_[round] + k * P + j);
    }
  iteration_indptr_.push_back((int)trees_.size());
}

// quantile_alpha on the device, uploaded when it differs from what the buffer holds
const float* Booster::upload_quantile_alpha(const std::vector<float>& alpha) {
  if (alpha != quantile_alpha_host_ || !quantile_alpha_dev_.p) {
    cudaStream_t s = engine_stream();
    quantile_alpha_dev_.alloc(std::max<size_t>(alpha.size(), 1));
    if (!alpha.empty()) CUDA_OK(cudaMemcpyAsync(quantile_alpha_dev_.p, alpha.data(), sizeof(float) * alpha.size(), cudaMemcpyHostToDevice, s));
    Comm::get().sync_stream(s);
    quantile_alpha_host_ = alpha;
  }
  return quantile_alpha_dev_.p;
}

void Booster::gradient_based_sample(const float2* src, float2* dst, int64_t gp_stride, int64_t n, int round, int j, unsigned* absmax) {
  GbsSampleArgs a{}; a.src = src; a.dst = dst; a.absmax = absmax; a.st = gbs_.st.p; a.gp_stride = gp_stride; a.n = n;
  a.row_offset = (int64_t)Comm::get().rank() << 40; a.K = param_.num_outputs(); a.seed = param_.seed; a.stream = row_stream(round, j);
  launch_gradient_based_sample(a, engine_stream());
}

// The objective's gradient pairs at `margin` into gpair ([K][gp_stride]), rows outside round `round`'s sample zeroed, max|g| and
// max h folded into absmax (nullptr: not taken).  dense_g (constant_hessian only): g alone, as float[gp_stride].  The survival
// objectives have their own kernels (survival.cu), reg:absoluteerror and reg:quantileerror theirs (adaptive.cu), which also write
// the residuals fl(y - m) into resid ([K][n]; nullptr: not written); every other objective runs gradient_kernel.
void Booster::launch_objective(DMatrix* dm, const float* margin, int round, float2* gpair, int64_t gp_stride, unsigned* absmax, float subsample,
                               bool dense_g, float* resid, bool per_target_absmax) {
  cudaStream_t s = engine_stream();
  const int64_t row_offset = (int64_t)Comm::get().rank() << 40;
  if (param_.num_target > 1) {               // multi-target: one pair per label element (multi_target.cu)
    B200_CHECK(!dense_g, "multi-target gradients are (g,h) pairs");
    MultiGradArgs ma{}; ma.margin = margin; ma.label = dm->d_labels.p; ma.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
    ma.gpair = gpair; ma.resid = resid; ma.absmax = absmax; ma.err = builder_->err.p; ma.n = dm->n; ma.row_offset = row_offset; ma.gp_stride = gp_stride;
    ma.T = param_.num_target; ma.objective = param_.objective; ma.per_target = per_target_absmax ? 1 : 0; ma.scale_pos_weight = param_.scale_pos_weight;
    ma.subsample = subsample; ma.aux = objective_aux(param_); ma.seed = param_.seed; ma.iter = (unsigned long long)round;
    launch_multi_target_gradient(ma, s);
    return;
  }
  if (param_.objective == kAbsoluteError) {
    AbsErrGradArgs aa{}; aa.margin = margin; aa.label = dm->d_labels.p; aa.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
    aa.gpair = gpair; aa.resid = resid; aa.absmax = absmax; aa.n = dm->n; aa.row_offset = row_offset; aa.subsample = subsample; aa.seed = param_.seed;
    aa.iter = (unsigned long long)round; aa.dense_g = dense_g ? 1 : 0;
    launch_abserr_gradient(aa, s);
    return;
  }
  if (param_.objective == kQuantileError) {
    QuantileGradArgs qa{}; qa.margin = margin; qa.label = dm->d_labels.p; qa.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
    qa.alpha = quantile_alpha_device(); qa.gpair = gpair; qa.resid = resid; qa.absmax = absmax; qa.n = dm->n; qa.row_offset = row_offset;
    qa.gp_stride = gp_stride; qa.subsample = subsample; qa.seed = param_.seed; qa.iter = (unsigned long long)round; qa.dense_g = dense_g ? 1 : 0;
    qa.Q = param_.num_outputs(); qa.per_target = per_target_absmax ? 1 : 0;
    launch_quantile_gradient(qa, s);
    return;
  }
  if (objective_is_rank(param_.objective)) {
    B200_CHECK(!dense_g, "the ranking objectives write (g,h) pairs");
    B200_CHECK(!param_.rank_unbiased, "lambdarank_unbiased=true (position debiasing) is not implemented on the CUDA hist path; a model trained with it loads and predicts");
    const RankGroups& rg = rank_groups(dm, objective_name_.c_str());
    RankGradArgs ra{}; ra.margin = margin; ra.label = dm->d_labels.p; ra.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
    // w_g * (groups / sum of w_g), both totals over every rank.  Every rank enters the all-reduce, with or without weights (an
    // empty shard has no groups), and all of them or none must have weights.
    double t[3] = {dm->n > 0 ? (double)rg.G : 0.0, 0.0, ra.weight ? 1.0 : 0.0};
    for (float w : dm->weights) t[1] += (double)w;
    if (Comm::get().distributed()) {
      dsum_.ensure(4);
      CUDA_OK(cudaMemcpyAsync(dsum_.p, t, sizeof t, cudaMemcpyHostToDevice, s));
      Comm::get().allreduce_sum_f64(dsum_.p, 3, s);
      CUDA_OK(cudaMemcpyAsync(t, dsum_.p, sizeof t, cudaMemcpyDeviceToHost, s));
      Comm::get().sync_stream(s);
      B200_CHECK(t[2] == 0.0 || t[2] == (double)Comm::get().world(), std::string(objective_name_) + ": every rank's DMatrix or none must have weights");
    }
    ra.wscale = t[2] > 0.0 && t[1] > 0.0 ? t[0] / t[1] : 1.0;
    ra.gpair = gpair; ra.absmax = absmax; ra.n = dm->n; ra.row_offset = row_offset; ra.subsample = subsample; ra.seed = param_.seed;
    ra.iter = (unsigned long long)round; ra.objective = param_.objective; ra.k = param_.rank_k; ra.exp_gain = param_.rank_exp_gain;
    ra.normalization = param_.rank_normalization; ra.score_normalization = param_.rank_score_normalization;
    ra.mean = param_.rank_mean; ra.pair_stream = kRankPairStream + ((uint64_t)round << 20);
    launch_rank_gradient(ra, rg, &rank_scratch_, s);
    return;
  }
  if (objective_is_survival(param_.objective)) {
    B200_CHECK(!dense_g, "the survival objectives write (g,h) pairs");
    SurvivalGradArgs sa{}; sa.margin = margin; sa.label = dm->d_labels.p; sa.lower = dm->d_label_lower.p; sa.upper = dm->d_label_upper.p;
    sa.weight = dm->weights.empty() ? nullptr : dm->d_weights.p; sa.gpair = gpair; sa.absmax = absmax; sa.n = dm->n; sa.row_offset = row_offset;
    sa.subsample = subsample; sa.seed = param_.seed; sa.iter = (unsigned long long)round; sa.dist = param_.aft_dist; sa.sigma = param_.aft_sigma;
    if (param_.objective == kAft) { launch_aft_gradient(sa, s); return; }
    if (!dm->cox_order.valid) cox_sort(dm->d_labels.p, dm->n, &dm->cox_order, &cox_scratch_, s);
    launch_cox_gradient(sa, dm->cox_order, &cox_scratch_, s);
    return;
  }
  GradArgs ga{}; ga.margin = margin; ga.label = dm->d_labels.p; ga.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
  ga.gpair = gpair; ga.gp_stride = gp_stride; ga.absmax = absmax; ga.err = builder_->err.p; ga.n = dm->n; ga.row_offset = row_offset; ga.K = param_.num_class;
  ga.objective = param_.objective; ga.scale_pos_weight = param_.scale_pos_weight; ga.subsample = subsample; ga.seed = param_.seed;
  ga.iter = (unsigned long long)round; ga.aux = objective_aux(param_); ga.dense_g = dense_g ? 1 : 0;
  launch_gradient(ga, s);
}

// dm's query groups on the device (one group of all rows without groups), built on first use; what (an objective or metric)
// reads one weight per group
const RankGroups& Booster::rank_groups(DMatrix* dm, const char* what) {
  check_labels(dm);
  B200_CHECK(dm->weights.empty() || (int64_t)dm->weights.size() == dm->num_groups(), std::string(what) + " reads one weight per query group: the DMatrix has " +
             std::to_string(dm->num_groups()) + " groups but " + std::to_string(dm->weights.size()) + " weights");
  if (!dm->rank_groups.valid) rank_groups_build(dm->group_ptr, dm->d_labels.p, dm->n, &dm->rank_groups, &rank_scratch_, engine_stream());
  return dm->rank_groups;
}

void Booster::debug_gradient(DMatrix* dm, const float* margin, int round, float* out) {
  configure();
  cudaStream_t s = engine_stream();
  if (param_.objective == kAft) check_aft_bounds(dm); else { check_targets(dm, true); check_labels(dm); }
  dm->ensure_binned(param_.max_bin); builder_for(dm);        // the builder owns the label-error flag gradient_kernel writes
  const int K = param_.num_outputs();
  const int64_t n = dm->n;
  DevBuf<float> d_margin; DevBuf<float2> d_gp; d_margin.alloc((size_t)n * K); d_gp.alloc((size_t)n * K);
  if (n) CUDA_OK(cudaMemcpyAsync(d_margin.p, margin, sizeof(float) * n * K, cudaMemcpyHostToDevice, s));
  const bool gbs = gradient_based_sampling();
  launch_objective(dm, d_margin.p, round, d_gp.p, n, nullptr, gbs ? 1.0f : param_.subsample, false, nullptr);      // always the (g,h) pairs
  if (gbs) {                 // the gradient-based sample of tree 0 of each class, as update_one_iter takes it
    gradient_based_threshold(d_gp.p, n, n, K, param_.subsample, &gbs_, s);
    gradient_based_sample(d_gp.p, d_gp.p, n, n, round, 0, nullptr);
  }
  std::vector<float2> h((size_t)n * K);
  if (n) CUDA_OK(cudaMemcpyAsync(h.data(), d_gp.p, sizeof(float2) * h.size(), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  for (int64_t r = 0; r < n; ++r)
    for (int k = 0; k < K; ++k) { out[(r * K + k) * 2] = h[(size_t)k * n + r].x; out[(r * K + k) * 2 + 1] = h[(size_t)k * n + r].y; }
}

// grow_policy=lossguide: expansions per tree = leaves - 1, bounded by max_leaves or by a full tree of max_depth
static int lossguide_iters(const TrainParam& p) {
  if (!p.lossguide) return 0;
  if (p.max_leaves > 0) return std::max(1, p.max_leaves - 1);
  return (1 << p.max_depth) - 1;
}

// a round's P trees of a class share its learning rate: leaves are fl(eta / P) * w (upstream BoostNewTrees); exact eta at P = 1
static TrainParamDev to_dev(const TrainParam& p) {
  TrainParamDev d; d.eta = p.eta / (float)p.num_parallel_tree; d.lambda = p.lambda; d.alpha = p.alpha; d.gamma = p.gamma; d.min_child_weight = p.min_child_weight;
  d.max_delta_step = p.max_delta_step; d.max_depth = p.max_depth; d.max_leaves = p.max_leaves; return d;
}

TreeBuilder& Booster::builder_for(DMatrix* dm) {
  builder_->ensure(dm->binned_view(), param_.max_depth, param_.num_outputs(), lossguide_iters(param_), (int)interaction_.size());
  return *builder_;
}

// Constant-hessian growth: every row has h == 1 in every round.  The round's gradients are then written as a dense float g
// (launch_objective) and the tree reads them so (root_mode != 0); this one predicate decides both.  B200XGB_NO_CONSTH turns it off.
bool Booster::constant_hessian(const DMatrix& dm) const {
  static const bool no_consth = getenv("B200XGB_NO_CONSTH") != nullptr;
  return !no_consth && (param_.objective == kSquaredError || param_.objective == kAbsoluteError || param_.objective == kQuantileError) &&
         param_.num_outputs() == 1 && dm.weights.empty() &&
         param_.subsample >= 1.0f && param_.scale_pos_weight == 1.0f;
}

// The only place TreeInputs are filled.  mask: the tree's column sets (empty = no column sampling), uploaded with its index;
// the constraints are uploaded here too.
TreeInputs Booster::tree_inputs(const DMatrix& dm, const std::string& mask, int tree_index, float* margin, int k) {
  TreeBuilder& b = *builder_;
  TreeInputs in{};                 // no padding bytes: every byte is zero before the fields are set
  in.bm = dm.binned_view(); in.cut_ptrs = dm.d_cut_ptrs.p; in.cut_vals = dm.d_cut_vals.p; in.min_vals = dm.d_min_vals.p;
  in.margin = margin; in.K = param_.num_outputs(); in.k = k;
  in.p = to_dev(param_); in.colsample_bynode = param_.colsample_bynode; in.seed = param_.seed; in.lg_iters = lossguide_iters(param_);
  in.mask = mask.empty() ? nullptr : b.upload_mask(mask, tree_index);
  in.monotone = b.upload_monotone(monotone_, dm.F);
  b.upload_interaction(interaction_, dm.F); in.n_ic = (int)interaction_.size();
  in.root_mode = !constant_hessian(dm) ? 0 : b.root_h_valid && b.root_h_uid == dm.uid && b.root_h_version == dm.binned_version ? 2 : 1;
  in.world = Comm::get().world();
  if (objective_is_adaptive(param_.objective)) {
    // output k's residual column and quantile
    in.resid = b.adapt.resid.p + (size_t)k * dm.n; in.alpha = param_.objective == kQuantileError ? param_.quantile_alpha[k] : 0.5f;
    in.adaptive = dm.weights.empty() ? 1 : gradient_based_sampling() ? 3 : 2;
    if (in.adaptive == 3) in.weight = dm.d_weights.p;
  }
  return in;
}

// One tree of class k: its column sets, the launch sequence, then the finished tree into the model.
void Booster::grow_one_tree(DMatrix* dtrain, PredCache& cache, int k, int tree_index) {
  cudaStream_t s = engine_stream();
  TreeBuilder& b = *builder_;
  std::string mask;
  if (param_.colsample_bytree < 1.0f || param_.colsample_bylevel < 1.0f || param_.colsample_bynode < 1.0f) {
    // one mask per level [max_depth][F]: bytree -> bylevel; bynode is applied inside eval_kernel
    const std::string tm = colsample_mask(param_.seed, tree_index, dtrain->F, param_.colsample_bytree);
    for (int d = 0; d < param_.max_depth; ++d) mask += subset_mask(tm, param_.colsample_bylevel, param_.seed, 0x300000ull + 64ull * (uint64_t)tree_index + (uint64_t)d);
  }
  const TreeInputs in = tree_inputs(*dtrain, mask, tree_index, cache.margin.p, k);
  b.grow(in);
  if (in.root_mode == 1) { b.root_h_valid = true; b.root_h_uid = dtrain->uid; b.root_h_version = dtrain->binned_version; }

  // ---- hand the finished tree to the model: device copy for prediction, async host copy for model IO
  reserve_nodes((size_t)b.cap_nodes, 64 * (size_t)b.cap_nodes);
  CUDA_OK(cudaMemcpyAsync(d_nodes.p + d_nodes_used, b.packed.p, sizeof(DevNode) * (size_t)b.cap_nodes, cudaMemcpyDeviceToDevice, s));
  if (pending_.size() - (size_t)std::count_if(pending_.begin(), pending_.end(), [](const PendingTree& p) { return p.staging == nullptr; }) >= 512) sync_model();
  const float weight = dart_.on ? dart_new_weight_ : 1.0f;
  append_device_tree(k, d_nodes_used, b.cap_nodes, b.stage_tree(), weight);
  d_nodes_used += (size_t)b.cap_nodes;
  d_trees_uploaded = 0;                      // offsets/info arrays need a refresh before the next predict
  cache.trees_applied = (int)trees_.size();  // update_margin_kernel already added this tree's leaves (times its weight) to the cache
  cache.weights.push_back(weight);
}

// ---------------------------------------------------------------------------------------------
// process_type=update (upstream GBTree::InitUpdater / BoostNewTrees with updater=refresh,prune; DESIGN.md "Refresh and prune")
// ---------------------------------------------------------------------------------------------
// The model's layers become the trees to update, packed on the device once; the model keeps base_score, num_feature,
// num_class and num_parallel_tree and nothing else, and every prediction cache starts over.
void Booster::begin_update() {
  cudaStream_t s = engine_stream();
  sync_model();
  UpdateState& u = *update_;
  u.trees = trees_; u.tree_info = tree_info_; u.indptr = iteration_indptr_;
  bool adjacent = true;
  for (size_t t = 0; t < u.trees.size(); ++t) {
    // the refresh walks the nodes reachable from the root as a tree: none of them may be the child of two of them
    const HostTree& h = u.trees[t];
    std::vector<char> reached((size_t)h.num_nodes(), 0); reached[0] = 1;
    for (int i = 0; i < h.num_nodes(); ++i) {
      if (!reached[i] || h.left[i] < 0) continue;
      B200_CHECK(!reached[h.left[i]] && !reached[h.right[i]], "process_type=update: tree " + std::to_string(t) + " is not a tree (a node of it has two parents)");
      reached[h.left[i]] = 1; reached[h.right[i]] = 1;
      if (h.right[i] != h.left[i] + 1) adjacent = false;
    }
  }
  reset_model();
  children_adjacent_ = adjacent;                   // the compaction keeps sibling pairs adjacent
  base_score_estimated_ = true;                    // never re-estimated: the trees to update were fitted on top of it
  const int nt = (int)u.trees.size();
  u.node_off.assign(nt + 1, 0); u.block_off.assign(nt, 0);
  int64_t blk = 0;
  for (int t = 0; t < nt; ++t) {
    const int nn = u.trees[t].num_nodes();
    u.node_off[t + 1] = u.node_off[t] + nn;
    u.block_off[t] = blk; blk += (int64_t)((tree_block_bytes((size_t)nn) + 255) & ~(size_t)255);
  }
  const size_t N = (size_t)u.node_off[nt];
  u.started = true;
  if (N == 0) return;
  std::vector<unsigned char> host(tree_block_bytes(N));
  const TreeArrays h = tree_block_layout(host.data(), N).t;
  std::vector<DevNode> dn(N);
  for (int t = 0; t < nt; ++t) {
    const HostTree& tr = u.trees[t];
    for (int i = 0; i < tr.num_nodes(); ++i) {
      const size_t j = (size_t)u.node_off[t] + i;
      h.left[j] = tr.left[i]; h.right[j] = tr.right[i]; h.parent[j] = tr.parent[i]; h.split_index[j] = tr.split_index[i];
      h.split_bin[j] = tr.split_bin[i]; h.default_left[j] = tr.default_left[i]; h.split_cond[j] = tr.split_cond[i];
      h.base_weight[j] = tr.base_weight[i]; h.loss_chg[j] = tr.loss_chg[i]; h.sum_hess[j] = tr.sum_hess[i];
      dn[j].cond = tr.split_cond[i]; dn[j].left = tr.left[i]; dn[j].right = tr.right[i];
      dn[j].fidx_dl = (unsigned)tr.split_index[i] | ((unsigned)tr.default_left[i] << 31);
    }
  }
  u.in_block.alloc(host.size()); u.nodes.alloc(N); u.d_node_off.alloc(nt + 1); u.d_class.alloc(nt); u.d_block_off.alloc(nt);
  u.sums.alloc(N); u.scratch.alloc(3 * N); u.out_blocks.alloc((size_t)blk);
  u.sums.zero(s);
  CUDA_OK(cudaMemcpyAsync(u.in_block.p, host.data(), host.size(), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(u.nodes.p, dn.data(), sizeof(DevNode) * N, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(u.d_node_off.p, u.node_off.data(), sizeof(int) * (nt + 1), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(u.d_class.p, u.tree_info.data(), sizeof(int) * nt, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(u.d_block_off.p, u.block_off.data(), sizeof(int64_t) * nt, cudaMemcpyHostToDevice, s));
  Comm::get().sync_stream(s);                     // the host copies go out of scope
}

// Update round r: the gradients at the margin of the layers refreshed so far, the per-node sums of layer r's trees over every
// row, then refresh / prune / compaction of each tree on the device, and the trees into the model as grown trees would go.
void Booster::refresh_one_iter(DMatrix* dtrain) {
  cudaStream_t s = engine_stream();
  B200_CHECK(!dart_.on, "process_type=update is not implemented for booster=dart");
  B200_CHECK(num_target_ == 1, "multi-target: process_type=update is not implemented for a model with num_target = " + std::to_string(num_target_));
  check_label_ranges(dtrain);
  if (!update_->started) begin_update();
  UpdateState& u = *update_;
  const int round = layers();
  B200_CHECK(round < u.layers(), "boosting rounds cannot exceed the previous training rounds under process_type=update (the model to update has " +
             std::to_string(u.layers()) + " rounds)");
  const int K = param_.num_outputs();
  const int t0 = u.indptr[round], t1 = u.indptr[round + 1], T = t1 - t0;
  for (int t = t0; t < t1; ++t) B200_CHECK(u.tree_info[t] >= 0 && u.tree_info[t] < K, "process_type=update: tree " + std::to_string(t) + " belongs to class " +
                                           std::to_string(u.tree_info[t]) + " but the model has " + std::to_string(K) + " outputs");
  // the fixed-point grid follows the rows of the whole job, as for growth (TreeBuilder::ensure): N GPUs and one agree
  if (u.global_n_uid != dtrain->uid || u.global_n == 0) {
    u.global_n = dtrain->n;
    if (Comm::get().distributed()) {
      DevBuf<double> dsum; dsum.alloc(1); double v = (double)dtrain->n;
      CUDA_OK(cudaMemcpyAsync(dsum.p, &v, sizeof v, cudaMemcpyHostToDevice, s));
      Comm::get().allreduce_sum_f64(dsum.p, 1, s);
      CUDA_OK(cudaMemcpyAsync(&v, dsum.p, sizeof v, cudaMemcpyDeviceToHost, s));
      Comm::get().sync_stream(s);
      u.global_n = (int64_t)v;
    }
    u.global_n_uid = dtrain->uid;
  }
  PredCache& cache = cache_for(dtrain);
  bring_cache_up_to_date(dtrain, cache);
  // every row's (g, h) pairs (the refresher uses every row: no row sampling) and the round's fixed-point scales
  const int64_t n = dtrain->n;
  u.gpair.ensure((size_t)std::max<int64_t>(n, 1) * K); u.absmax.ensure(2); u.scales.ensure(4);
  if (!builder_->err.p) { builder_->err.alloc(1); builder_->err.zero(s); }     // the label-error flag gradient_kernel writes
  CUDA_OK(cudaMemsetAsync(u.absmax.p, 0, 8, s));
  launch_objective(dtrain, cache.margin.p, round, u.gpair.p, n, u.absmax.p, 1.0f, false, nullptr);
  Comm::get().allreduce_max_u32(u.absmax.p, 2, s);
  GrowState gs{}; gs.absmax = u.absmax.p; gs.scales = u.scales.p;
  launch_scales(gs, grad_bits_for(u.global_n), s);
  // the layer's leaf sums, exact int64, all-reduced over the ranks
  const int base = u.node_off[t0], nl = u.node_off[t1] - base;
  const size_t N = (size_t)u.node_off.back();
  CUDA_OK(cudaMemsetAsync(u.sums.p + base, 0, sizeof(GH64) * nl, s));
  RefreshSumArgs sa{}; sa.X = dtrain->X.p; sa.n = n; sa.F = dtrain->F; sa.nodes = u.nodes.p; sa.tree_node_off = u.d_node_off.p + t0;
  sa.tree_class = u.d_class.p + t0; sa.T = T; sa.layer_nodes = nl; sa.gpair = u.gpair.p; sa.gp_stride = n; sa.scales = u.scales.p; sa.sums = u.sums.p;
  launch_refresh_sums(sa, s);
  Comm::get().allreduce_sum_i64(u.sums.p + base, 2 * (size_t)nl, s);
  // refresh / prune / compaction, straight into the device model and the trees' blocks
  reserve_nodes((size_t)nl, 64 * (size_t)nl);
  RefreshTreeArgs ta{}; ta.in = tree_block_layout(u.in_block.p, N).t; ta.tree_node_off = u.d_node_off.p + t0; ta.T = T; ta.sums = u.sums.p;
  ta.scales = u.scales.p; ta.p = to_dev(param_); ta.nops = (int)update_ops_.size();
  for (int i = 0; i < ta.nops; ++i) ta.ops[i] = update_ops_[i];
  ta.refresh_leaf = refresh_leaf_; ta.scratch = u.scratch.p; ta.total_nodes = (int64_t)N; ta.out_blocks = u.out_blocks.p; ta.block_off = u.d_block_off.p;
  ta.first_tree = t0; ta.out_nodes = d_nodes.p + d_nodes_used;
  launch_refresh_trees(ta, s);
  TreeBuilder& b = *builder_;
  for (int t = t0; t < t1; ++t) {
    const size_t nn = (size_t)u.trees[t].num_nodes();
    if (pending_.size() - (size_t)std::count_if(pending_.begin(), pending_.end(), [](const PendingTree& p) { return p.staging == nullptr; }) >= 512) sync_model();
    PendingTree pt; pt.cap_nodes = nn; pt.staging = b.pinned.take(tree_block_bytes(nn));
    if (!b.free_events.empty()) { pt.ready = b.free_events.back(); b.free_events.pop_back(); }
    else CUDA_OK(cudaEventCreateWithFlags(&pt.ready, cudaEventDisableTiming));
    CUDA_OK(cudaMemcpyAsync(pt.staging, u.out_blocks.p + u.block_off[t], tree_block_bytes(nn), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaEventRecord(pt.ready, s));
    append_device_tree(u.tree_info[t], d_nodes_used + (size_t)(u.node_off[t] - base), (int)nn, pt, 1.0f);
  }
  d_nodes_used += (size_t)nl;
  d_trees_uploaded = 0;                      // offsets/info arrays need a refresh before the next predict
  iteration_indptr_.push_back((int)trees_.size());
}

void Booster::debug_refresh_sums(std::vector<long long>* out) {
  const UpdateState& u = *update_;
  const size_t N = u.node_off.empty() ? 0 : (size_t)u.node_off.back();
  out->assign(2 * N, 0);
  if (N == 0 || !u.sums.p) return;
  cudaStream_t s = engine_stream();
  CUDA_OK(cudaMemcpyAsync(out->data(), u.sums.p, sizeof(GH64) * N, cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
}

void Booster::boost_one_iter(DMatrix*, const float*, const float*, size_t) {
  throw Error("custom objective (BoostOneIter) is not implemented on the CUDA hist path");
}

int Booster::boosted_rounds() { configure(); return layers(); }

// ---------------------------------------------------------------------------------------------
// evaluation  (upstream src/learner.cc EvalOneIter: "[iter]\t<name>-<metric>:<value>")
// ---------------------------------------------------------------------------------------------
static std::string default_metric(const TrainParam& p) {
  switch (p.objective) {
    case kSquaredError: case kRegLogistic: return "rmse";
    case kAbsoluteError: return "mae";
    case kQuantileError: return "quantile";
    case kBinaryLogistic: case kLogitRaw: return "logloss";
    case kSquaredLogError: return "rmsle";
    case kPseudoHuber: return "mphe";
    case kPoisson: return "poisson-nloglik";
    case kGamma: return "gamma-nloglik";
    case kTweedie: { char buf[64]; snprintf(buf, sizeof buf, "tweedie-nloglik@%g", (double)p.tweedie_variance_power); return buf; }
    case kHinge: return "error";
    case kAft: return "aft-nloglik";
    case kCox: return "cox-nloglik";
    case kRankPairwise: case kRankNdcg: return p.rank_mean ? "ndcg" : "ndcg@" + std::to_string(p.rank_k);
    case kRankMap: return p.rank_mean ? "map" : "map@" + std::to_string(p.rank_k);
    default: return "mlogloss";
  }
}

// ndcg, ndcg@k, ndcg-, ndcg@k-, map, map@k, map-, map@k- (k = 0: the whole group; '-' scores a group without relevant documents 0)
static bool parse_rank_metric(const std::string& name, int* map, int* k, int* minus) {
  std::string s = name;
  if (s.rfind("ndcg", 0) == 0) { *map = 0; s = s.substr(4); }
  else if (s.rfind("map", 0) == 0 && (s.size() == 3 || s[3] == '@' || s[3] == '-')) { *map = 1; s = s.substr(3); }
  else return false;
  *minus = 0; *k = 0;
  if (!s.empty() && s.back() == '-') { *minus = 1; s.pop_back(); }
  if (s.empty()) return true;
  B200_CHECK(s[0] == '@' && s.size() > 1 && s.find_first_not_of("0123456789", 1) == std::string::npos && s.size() < 11,
             "Invalid ranking metric " + name + " (ndcg, ndcg@k, ndcg-, ndcg@k-, map, map@k, map-, map@k-)");
  *k = std::stoi(s.substr(1));
  B200_CHECK(*k >= 1, "Invalid ranking metric " + name + ": k must be >= 1");
  return true;
}

std::string Booster::eval_one_iter(int iter, const std::vector<DMatrix*>& dms, const std::vector<std::string>& names) {
  configure();
  cudaStream_t s = engine_stream();
  std::vector<std::string> metrics = eval_metrics_;
  if (metrics.empty()) metrics.push_back(default_metric(param_));
  dsum_.ensure(4);
  std::string out = "[" + std::to_string(iter) + "]";
  for (size_t i = 0; i < dms.size(); ++i) {
    DMatrix* dm = dms[i];
    if (param_.objective != kAft) { check_targets(dm, false); check_labels(dm); }
    PredCache& c = cache_for(dm);
    bring_cache_up_to_date(dm, c);
    for (const std::string& mname : metrics) {
      MetricArgs ma{}; ma.margin = c.margin.p; ma.label = dm->d_labels.p; ma.weight = dm->weights.empty() ? nullptr : dm->d_weights.p;
      ma.out = dsum_.p; ma.n = dm->n; ma.K = param_.num_class; ma.threshold = 0.5f;
      ma.is_logistic = (param_.objective == kBinaryLogistic || param_.objective == kRegLogistic) ? 1 : 0;
      ma.transform = objective_transform(param_.objective); ma.aux = 0.0f;
      std::string base = mname;
      if (mname.rfind("tweedie-nloglik@", 0) == 0) { base = "tweedie-nloglik"; ma.aux = std::stof(mname.substr(16)); B200_CHECK(ma.aux >= 1.0f && ma.aux < 2.0f, "tweedie variance power must be in interval [1, 2)"); }
      if (mname.rfind("error@", 0) == 0) { base = "error"; ma.threshold = std::stof(mname.substr(6)); }
      // multi-target: the element-wise metrics over the n x T elements; auc / aucpr raise below as for any model with several outputs
      static const std::map<std::string, int> kElementwise = {{"rmse", kMetricRmse}, {"rmsle", kMetricRmsle}, {"mae", kMetricMae}, {"mape", kMetricMape},
                                                             {"mphe", kMetricMphe}, {"logloss", kMetricLogloss}, {"error", kMetricError}};
      const auto ew = kElementwise.find(base);
      if (param_.num_target > 1)
        B200_CHECK(ew != kElementwise.end() || base == "auc" || base == "aucpr", "multi-target: metric " + mname + " is not implemented for a model with " +
                   std::to_string(param_.num_target) + " targets (rmse, rmsle, mae, mape, mphe, logloss, error and error@t are)");
      int rank_map = 0, rank_k = 0, rank_minus = 0;
      if (parse_rank_metric(mname, &rank_map, &rank_k, &rank_minus)) {     // ndcg / map over the query groups (rank.cu)
        const RankGroups& rg = rank_groups(dm, mname.c_str());
        rank_metric(c.margin.p, dm->d_labels.p, ma.weight, rg, rank_map, rank_k, param_.rank_exp_gain, rank_minus, &rank_scratch_, dsum_.p, s);
        Comm::get().allreduce_sum_f64(dsum_.p, 2, s);
        double h[2];
        CUDA_OK(cudaMemcpyAsync(h, dsum_.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
        Comm::get().sync_stream(s);
        char buf[64]; snprintf(buf, sizeof buf, "%.17g", h[1] > 0.0 ? h[0] / h[1] : 0.0);
        out += "\t" + names[i] + "-" + mname + ":" + buf;
        continue;
      }
      B200_CHECK(mname.rfind("pre@", 0) != 0 && mname != "pre", "metric " + mname + ": the pre / pre@k ranking metric is not implemented on the CUDA hist path (ndcg and map are)");
      check_row_weights(dm);
      const bool multiclass = (param_.objective == kSoftprob || param_.objective == kSoftmax) && param_.num_class > 1;
      if (base == "aucpr" || (base == "auc" && multiclass)) {
        // curve.cu: binary aucpr, and auc / aucpr one-vs-rest over the softmax probabilities (DESIGN.md "AUC family")
        check_labels(dm);                        // survival:aft skips the check above; its matrices may carry bounds only
        B200_CHECK(!objective_is_rank(param_.objective) || dm->group_ptr.empty(), mname + " under a rank:* objective on a DMatrix with query groups (ranking " +
                   (base == "auc" ? "AUC" : "PR-AUC") + ") is not implemented on the CUDA hist path");
        B200_CHECK(multiclass || param_.num_outputs() <= 1, mname + " reads one output per row or the softmax probabilities of multi:softprob / multi:softmax; a " +
                   objective_name_ + " model with " + std::to_string(param_.num_outputs()) + " outputs per row is not supported");
        const int pr = base == "aucpr" ? 1 : 0, K = multiclass ? param_.num_class : 0;
        const int logistic = (param_.objective == kBinaryLogistic || param_.objective == kRegLogistic) ? 1 : 0;
        const int len = curve_metric_local(c.margin.p, dm->d_labels.p, ma.weight, dm->n, K, logistic, pr, &curve_scratch_, s);
        Comm::get().allreduce_sum_f64(curve_scratch_.vec.p, len, s);
        curve_metric_finish(K, pr, Comm::get().world(), &curve_scratch_, dsum_.p, s);
        double h[4];
        CUDA_OK(cudaMemcpyAsync(h, dsum_.p, 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
        Comm::get().sync_stream(s);
        if (pr && !K) {
          B200_CHECK(h[3] == 0.0, "Check failed: label must be in [0, 1] for aucpr (binary PR-AUC reads the label as the positive share of a row)");
          B200_CHECK(h[1] > 0.0 && h[2] > 0.0, "Check failed: !auc_error AUC: the dataset only contains pos or neg samples");
        }
        char buf[64]; snprintf(buf, sizeof buf, "%.17g", h[0]);
        out += "\t" + names[i] + "-" + mname + ":" + (std::isnan(h[0]) ? std::string("nan") : std::string(buf));
        continue;
      }
      if (base == "auc") {
        // validated on hardware against sklearn.metrics.roc_auc_score (tests/test_gpu_parity.py::test_auc_matches_sklearn)
        check_labels(dm);                        // survival:aft skips the check above; its matrices may carry bounds only
        B200_CHECK(param_.num_outputs() <= 1, "auc reads one output per row or the softmax probabilities of multi:softprob / multi:softmax; a " +
                   objective_name_ + " model with " + std::to_string(param_.num_outputs()) + " outputs per row is not supported");
        B200_CHECK(!objective_is_rank(param_.objective) || dm->group_ptr.empty(), "auc under a rank:* objective on a DMatrix with query groups (ranking AUC) is not implemented on the CUDA hist path");
        const int logistic = (param_.objective == kBinaryLogistic || param_.objective == kRegLogistic) ? 1 : 0;
        compute_auc_device(c.margin.p, dm->d_labels.p, dm->weights.empty() ? nullptr : dm->d_weights.p, dm->n, logistic, dsum_.p, s);
        double h3[3];
        CUDA_OK(cudaMemcpyAsync(h3, dsum_.p, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
        Comm::get().sync_stream(s);
        double pair[2] = {h3[0], h3[1] * h3[2]};
        if (Comm::get().distributed()) {
          CUDA_OK(cudaMemcpyAsync(dsum_.p, pair, 2 * sizeof(double), cudaMemcpyHostToDevice, s));
          Comm::get().allreduce_sum_f64(dsum_.p, 2, s);
          CUDA_OK(cudaMemcpyAsync(pair, dsum_.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
          Comm::get().sync_stream(s);
        }
        B200_CHECK(pair[1] > 0.0, "Check failed: !auc_error AUC: the dataset only contains pos or neg samples");
        char buf[64]; snprintf(buf, sizeof buf, "%.17g", pair[0] / pair[1]);
        out += "\t" + names[i] + "-" + mname + ":" + buf;
        continue;
      }
      if (param_.num_target > 1) {               // sum_i sum_j w_i loss(y_ij, p_ij) / (T sum_i w_i) (multi_target.cu)
        MultiMetricArgs mt{}; mt.margin = c.margin.p; mt.label = dm->d_labels.p; mt.weight = ma.weight; mt.out = dsum_.p; mt.n = dm->n; mt.T = param_.num_target;
        mt.metric = ew->second; mt.is_logistic = ma.is_logistic || (param_.objective == kLogitRaw && (ew->second == kMetricLogloss || ew->second == kMetricError));
        mt.transform = ma.transform; mt.threshold = ma.threshold; mt.aux = ew->second == kMetricMphe ? param_.huber_slope : 0.0f;
        CUDA_OK(cudaMemsetAsync(dsum_.p, 0, 2 * sizeof(double), s));
        launch_multi_target_metric(mt, s);
      } else if (mname == "aft-nloglik" || mname == "interval-regression-accuracy") {     // at the margin, in double (survival.cu)
        check_aft_bounds(dm);
        CUDA_OK(cudaMemsetAsync(dsum_.p, 0, 2 * sizeof(double), s));
        launch_aft_metric(c.margin.p, dm->d_label_lower.p, dm->d_label_upper.p, ma.weight, dm->n, param_.aft_dist, param_.aft_sigma,
                          mname == "aft-nloglik" ? 0 : 1, dsum_.p, s);
      } else if (mname == "cox-nloglik") {        // unweighted, per event, with the deterministic risk-set sums of survival:cox
        B200_CHECK(!Comm::get().distributed(), "cox-nloglik is not supported with more than one GPU (world_size > 1)");
        check_labels(dm);
        if (!dm->cox_order.valid) cox_sort(dm->d_labels.p, dm->n, &dm->cox_order, &cox_scratch_, s);
        cox_nloglik(c.margin.p, dm->n, dm->cox_order, &cox_scratch_, dsum_.p, s);
      } else if (mname == "quantile") {           // pinball loss of every output at its quantile_alpha entry (adaptive.cu)
        check_labels(dm);
        B200_CHECK(!param_.quantile_alpha.empty() || raw_params_.count("quantile_alpha"), "the quantile metric needs the parameter quantile_alpha");
        const std::vector<float> alpha = param_.objective == kQuantileError ? param_.quantile_alpha : parse_quantile_alpha(raw_params_.at("quantile_alpha"));
        B200_CHECK((int)alpha.size() == param_.num_outputs(), "the quantile metric: the model has " + std::to_string(param_.num_outputs()) +
                   " outputs per row but quantile_alpha has " + std::to_string(alpha.size()) + " values");
        CUDA_OK(cudaMemsetAsync(dsum_.p, 0, 2 * sizeof(double), s));
        launch_quantile_metric(c.margin.p, dm->d_labels.p, ma.weight, upload_quantile_alpha(alpha), (int)alpha.size(), dm->n, dsum_.p, s);
      } else {
        if (param_.objective == kAft) check_labels(dm);
        B200_CHECK(param_.objective != kQuantileError || param_.num_outputs() == 1, "metric " + mname + " reads one output per row; a reg:quantileerror model with " +
                   std::to_string(param_.num_outputs()) + " outputs is evaluated with the quantile metric");
        if (base == "rmse") ma.metric = kMetricRmse; else if (base == "mse") ma.metric = kMetricRmse; else if (base == "mae") ma.metric = kMetricMae;
        else if (base == "logloss") ma.metric = kMetricLogloss; else if (base == "error") ma.metric = kMetricError;
        else if (base == "merror") ma.metric = kMetricMerror; else if (base == "mlogloss") ma.metric = kMetricMlogloss;
        else if (base == "rmsle") ma.metric = kMetricRmsle; else if (base == "mape") ma.metric = kMetricMape;
        else if (base == "mphe") { ma.metric = kMetricMphe; ma.aux = param_.huber_slope; }
        else if (base == "poisson-nloglik") ma.metric = kMetricPoissonNll; else if (base == "gamma-nloglik") ma.metric = kMetricGammaNll;
        else if (base == "gamma-deviance") ma.metric = kMetricGammaDeviance;
        else if (base == "tweedie-nloglik") { ma.metric = kMetricTweedieNll; if (ma.aux == 0.0f) throw Error("tweedie-nloglik needs its variance power: tweedie-nloglik@rho"); }
        else throw Error("Unknown metric function " + mname + " (the CUDA hist path implements rmse, mse, rmsle, mae, quantile, mape, mphe, logloss, error, error@t, merror, mlogloss, auc, aucpr, poisson-nloglik, gamma-nloglik, gamma-deviance, tweedie-nloglik@rho, aft-nloglik, interval-regression-accuracy, cox-nloglik, ndcg, ndcg@k, map, map@k)");
        if (param_.objective == kLogitRaw && (ma.metric == kMetricLogloss || ma.metric == kMetricError)) ma.is_logistic = 1;
        if ((ma.metric == kMetricMerror || ma.metric == kMetricMlogloss)) B200_CHECK(param_.num_class > 1, "Check failed: preds.size() == info.labels_.size() : label and prediction size not match, hint: use merror or mlogloss for multi-class classification");
        CUDA_OK(cudaMemsetAsync(dsum_.p, 0, 2 * sizeof(double), s));
        launch_metric(ma, s);
      }
      Comm::get().allreduce_sum_f64(dsum_.p, 2, s);
      double h[2];
      CUDA_OK(cudaMemcpyAsync(h, dsum_.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
      Comm::get().sync_stream(s);
      double v = h[1] == 0.0 ? h[0] : h[0] / h[1];
      if (mname == "rmse" || mname == "rmsle") v = std::sqrt(v);
      if (mname == "gamma-deviance") v *= 2.0;
      char buf[64]; snprintf(buf, sizeof buf, "%.17g", v);
      out += "\t" + names[i] + "-" + mname + ":" + buf;
    }
  }
  return out;
}

// The container's custom_metrics (DESIGN.md "Container metrics"): what the device pass decides exactly, in the raw form the
// Python finisher turns into scikit-learn's values; anything left undecided is evaluated by the container's own function.
void Booster::eval_container_metrics(DMatrix* dm, const std::vector<std::string>& names, bool output_margin, long long* out) {
  configure();
  static const char* kClass[] = {"accuracy", "balanced_accuracy", "f1", "f1_binary", "f1_macro", "precision", "precision_macro",
                                 "precision_micro", "recall", "recall_macro", "recall_micro"};
  bool want_class = false, want_reg = false, want_r2 = false;
  for (const std::string& name : names) {
    if (std::find(std::begin(kClass), std::end(kClass), name) != std::end(kClass)) want_class = true;
    else if (name == "mse" || name == "rmse" || name == "mae") want_reg = true;
    else if (name == "r2") want_reg = want_r2 = true;
    else throw Error("unknown container metric " + name);
  }
  const int K = param_.num_outputs();
  const int cols = (!output_margin && param_.objective == kSoftmax) ? 1 : K;
  const int P = cols == 1 ? 2 : cols;
  const int64_t n = dm->n;
  std::fill(out, out + kContainerOutLen, 0LL);
  out[1] = n; out[2] = P; out[3] = kContainerLabels;
  if (n == 0 || dm->labels.size() != (size_t)n || param_.num_target > 1) return;      // a multi-target model: the container's own function
  want_class = want_class && P <= kContainerLabels;
  want_reg = want_reg && cols == 1 && n <= INT_MAX;
  want_r2 = want_r2 && want_reg;
  if (!want_class && !want_reg) return;
  cudaStream_t s = engine_stream();
  const float* margin;
  if (dart_.on) {
    // the dart cache carries each round's weight changes as fl(w_now - w_applied) * leaf, while predict() sums
    // fl(w_t * leaf_t) afresh: the two differ in the last bits, so the metrics read predict()'s own margins
    predict_margin(dm, 0, (int)trees_.size());
    margin = pred_margin_.p;
  } else {
    PredCache& c = cache_for(dm);
    bring_cache_up_to_date(dm, c);
    margin = c.margin.p;
  }
  ContainerArgs a{}; a.margin = margin; a.label = dm->d_labels.p; a.n = n; a.K = K;
  a.objective = param_.objective; a.output_margin = output_margin ? 1 : 0;
  a.want_class = want_class; a.want_reg = want_reg; a.want_r2 = want_r2;
  container_metrics_device(a, &dm->container_sums, &container_scratch_, s);
  const size_t len = kContainerOutHead + (size_t)kContainerLabels * P;
  CUDA_OK(cudaMemcpyAsync(out + 4, container_scratch_.out.p + 4, sizeof(long long) * (len - 4), cudaMemcpyDeviceToHost, s));
  long long bad = 0;
  CUDA_OK(cudaMemcpyAsync(&bad, container_scratch_.out.p, sizeof(long long), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  out[0] = (want_class && !(bad & 1) ? kDecidedClass : 0) | (want_reg && !(bad & 2) ? kDecidedReg : 0) |
           (want_r2 && !(bad & 2) ? kDecidedLabelSums : 0);
}

// ---------------------------------------------------------------------------------------------
// prediction (upstream Booster.predict -> XGBoosterPredictFromDMatrix; cpu_predictor.cc semantics)
// type: 0 value, 1 margin, 6 leaf
// ---------------------------------------------------------------------------------------------
void Booster::predict_margin(DMatrix* dm, int tb, int te) {
  cudaStream_t s = engine_stream();
  const int K = param_.num_outputs();
  const int64_t n = dm->n;
  upload_model();
  DevBuf<float>& margin = pred_margin_; margin.ensure((size_t)n * K);          // scratch kept across calls: no cudaMalloc / cudaFree per request
  if (!dm->base_margin.empty()) {
    B200_CHECK(dm->base_margin.size() == (size_t)n * K, "base_margin size does not match rows x groups");
    CUDA_OK(cudaMemcpyAsync(margin.p, dm->d_base_margin.p, sizeof(float) * n * K, cudaMemcpyDeviceToDevice, s));
  } else launch_fill(margin.p, n * K, base_margin(), s);
  if (dart_.on) {            // booster=dart: base + sum_t fl(w_t * leaf_t) in tree order (training=True predicts the same)
    dm->require_raw("booster=dart");
    std::vector<int> ids; std::vector<float> coef;
    for (int t = tb; t < te; ++t) { ids.push_back(t); coef.push_back(weight_drop_[t]); }
    if (!ids.empty()) dart_margin(dm, ids, coef, {}, margin.p, nullptr);
  } else {
    PredictArgs pa = predict_args(dm, tb, te);
    pa.margin = margin.p; pa.leaf = nullptr;
    run_predict(dm, pa, s);
  }
}

void Booster::predict(DMatrix* dm, int type, bool training, int iter_begin, int iter_end, bool strict_shape,
                      std::vector<float>* out, std::vector<uint64_t>* shape) {
  configure();
  (void)training;
  cudaStream_t s = engine_stream();
  const int K = param_.num_outputs();
  const int rounds = layers();
  if (iter_end == 0) iter_end = rounds;
  B200_CHECK(iter_begin >= 0 && iter_begin <= iter_end && iter_end <= rounds, "Invalid iteration range: [" + std::to_string(iter_begin) + ", " + std::to_string(iter_end) + ") for a model with " + std::to_string(rounds) + " rounds");
  if (num_feature_ > 0 && !trees_.empty())
    B200_CHECK(dm->F <= num_feature_ || true, "feature count mismatch");
  B200_CHECK(type == 0 || type == 1 || type == 2 || type == 6, "predict type " + std::to_string(type) + " (approximate contributions / interactions) is not implemented on the CUDA path");
  const int tb = iteration_indptr_[iter_begin], te = iteration_indptr_[iter_end];
  if (type == 2) { predict_contribs(dm, tb, te, out, shape); return; }
  upload_model();
  const int64_t n = dm->n;
  PredictArgs pa = predict_args(dm, tb, te);
  if (type == 6) {
    const int nt = te - tb;
    DevBuf<int>& leaf = pred_leaf_; leaf.ensure((size_t)n * std::max(nt, 1));
    pa.margin = nullptr; pa.leaf = leaf.p;
    run_predict(dm, pa, s);
    std::vector<int> h((size_t)n * nt);
    if (!h.empty()) CUDA_OK(cudaMemcpyAsync(h.data(), leaf.p, sizeof(int) * h.size(), cudaMemcpyDeviceToHost, s));
    Comm::get().sync_stream(s);
    out->resize(h.size());
    for (size_t i = 0; i < h.size(); ++i) (*out)[i] = (float)h[i];
    shape->assign({(uint64_t)n, (uint64_t)nt});
    return;
  }
  DevBuf<float>& margin = pred_margin_;
  predict_margin(dm, tb, te);
  int out_cols = K;
  DevBuf<float>& cls = pred_cls_;
  if (type == 0) {
    if (param_.objective == kSoftmax) { cls.ensure(n); launch_transform(margin.p, n, K, param_.objective, cls.p, s); out_cols = 1; }
    else if (param_.objective == kSoftprob) launch_transform(margin.p, n, K, param_.objective, nullptr, s);
    else launch_transform(margin.p, n * K, 1, param_.objective, nullptr, s);       // element-wise over the n x K outputs
  }
  out->resize((size_t)n * out_cols);
  if (!out->empty()) CUDA_OK(cudaMemcpyAsync(out->data(), (type == 0 && param_.objective == kSoftmax) ? cls.p : margin.p, sizeof(float) * out->size(), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  if (out_cols == 1 && !strict_shape) shape->assign({(uint64_t)n});
  else shape->assign({(uint64_t)n, (uint64_t)out_cols});
}

void Booster::debug_build_root_hist(DMatrix* dm, const float* gpair_host, std::vector<long long>* hist_out, float* scales_out,
                                    int repeats, float* ms_out, int mode, const unsigned* row_ids, int64_t n_ids) {
  configure(); dm->ensure_binned(param_.max_bin);
  builder_for(dm).debug_build_root_hist(dm->binned_view(), gpair_host, hist_out, scales_out, repeats, ms_out, mode, row_ids, n_ids);
}

// feat_mask (F bytes, nullptr = all) is the tree's column set
std::string Booster::debug_eval_root(DMatrix* dm, const long long* hist_fm, long long G, long long H, float max_g, float max_h,
                                     float lower, float upper, const unsigned char* feat_mask) {
  configure(); check_train_width(dm);
  B200_CHECK(interaction_.empty(), "debug_eval_root: interaction constraints are not supported");
  dm->ensure_binned(param_.max_bin); TreeBuilder& b = builder_for(dm); std::string mask;
  if (feat_mask || param_.colsample_bynode < 1.0f) mask = feat_mask ? std::string((const char*)feat_mask, (size_t)dm->F) : std::string((size_t)dm->F, (char)1);
  return b.debug_eval_root(tree_inputs(*dm, mask, 0, nullptr, 0), hist_fm, G, H, max_g, max_h, lower, upper);
}

// pred_contribs: path-dependent Tree SHAP on the device (shap.cu); output [n][F + 1], or [n][K][F + 1] for multi-class models
void Booster::predict_contribs(DMatrix* dm, int tb, int te, std::vector<float>* out, std::vector<uint64_t>* shape) {
  dm->require_raw("pred_contribs (SHAP)");
  cudaStream_t s = engine_stream();
  sync_model();
  const int K = param_.num_outputs();
  const int64_t n = dm->n;
  const int F = std::max(dm->F, num_feature_);
  B200_CHECK(dm->F == F, "pred_contribs: the data has " + std::to_string(dm->F) + " columns, the model uses " + std::to_string(F));
  std::vector<ShapNode> nodes; std::vector<int64_t> offs; std::vector<int> info;
  int max_depth = 0;
  for (int t = tb; t < te; ++t) {
    const HostTree& h = trees_[t];
    const int nn = h.num_nodes();
    const size_t base = nodes.size();
    offs.push_back((int64_t)base); info.push_back(tree_info_[t]);
    nodes.resize(base + nn);
    std::vector<int> depth(nn, 0);
    for (int i = 0; i < nn; ++i) {
      ShapNode& d = nodes[base + i];
      d.cond = h.split_cond[i]; d.left = h.left[i]; d.right = h.right[i]; d.fidx_dl = (unsigned)h.split_index[i] | ((unsigned)h.default_left[i] << 31);
      d.sum_hess = h.sum_hess[i]; d.mean = 0.0f;
      if (h.left[i] >= 0) { B200_CHECK(h.left[i] > i && h.right[i] > i, "pred_contribs: children must follow their parent in the node array"); depth[h.left[i]] = depth[h.right[i]] = depth[i] + 1; }
      max_depth = std::max(max_depth, depth[i]);
    }
    // cover-weighted mean value per node, children before parents (upstream FillNodeMeanValues, float arithmetic)
    for (int i = nn - 1; i >= 0; --i) {
      ShapNode& d = nodes[base + i];
      if (d.left < 0) d.mean = d.cond;
      else { float r = nodes[base + d.left].mean * nodes[base + d.left].sum_hess; r += nodes[base + d.right].mean * nodes[base + d.right].sum_hess; d.mean = r / d.sum_hess; }
    }
  }
  DevBuf<ShapNode> d_sn; DevBuf<int64_t> d_off; DevBuf<int> d_info; DevBuf<float> d_out, d_w;
  if (dart_.on && te > tb) {
    d_w.alloc((size_t)(te - tb));
    CUDA_OK(cudaMemcpyAsync(d_w.p, weight_drop_.data() + tb, sizeof(float) * (te - tb), cudaMemcpyHostToDevice, s));
  }
  d_sn.alloc(std::max<size_t>(nodes.size(), 1)); d_off.alloc(std::max<size_t>(offs.size(), 1)); d_info.alloc(std::max<size_t>(info.size(), 1));
  const size_t total = (size_t)n * K * (F + 1);
  d_out.alloc(std::max<size_t>(total, 1));
  if (!nodes.empty()) {
    CUDA_OK(cudaMemcpyAsync(d_sn.p, nodes.data(), sizeof(ShapNode) * nodes.size(), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(d_off.p, offs.data(), sizeof(int64_t) * offs.size(), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(d_info.p, info.data(), sizeof(int) * info.size(), cudaMemcpyHostToDevice, s));
  }
  CUDA_OK(cudaMemsetAsync(d_out.p, 0, sizeof(float) * std::max<size_t>(total, 1), s));
  ShapArgs sa{}; sa.X = dm->X.p; sa.n = n; sa.F = F; sa.nodes = d_sn.p; sa.tree_offset = d_off.p; sa.tree_info = d_info.p; sa.tree_begin = tb; sa.tree_end = te; sa.K = K;
  sa.out = d_out.p; sa.base_margin = base_margin(); sa.tree_weight = d_w.p;
  if (!dm->base_margin.empty()) { B200_CHECK(dm->base_margin.size() == (size_t)n * K, "base_margin size does not match rows x groups"); sa.base_margin_rows = dm->d_base_margin.p; }
  launch_shap(sa, max_depth, s);
  out->resize(total);
  if (total) CUDA_OK(cudaMemcpyAsync(out->data(), d_out.p, sizeof(float) * total, cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  if (K > 1) shape->assign({(uint64_t)n, (uint64_t)K, (uint64_t)(F + 1)}); else shape->assign({(uint64_t)n, (uint64_t)(F + 1)});
}

PredictArgs Booster::predict_args(DMatrix* dm, int tree_begin, int tree_end) {
  PredictArgs pa{}; pa.X = dm->X.p; pa.n = dm->n; pa.F = dm->F; pa.nodes = d_nodes.p; pa.tree_offset = d_tree_offset.p; pa.tree_info = d_tree_info.p;
  pa.tree_begin = tree_begin; pa.tree_end = tree_end; pa.K = param_.num_outputs(); pa.margin = nullptr; pa.leaf = nullptr;
  pa.h_tree_offset = h_tree_offset.data(); pa.has_nan = dm->has_missing ? 1 : 0; pa.children_adjacent = children_adjacent_ ? 1 : 0;
  pa.model_F = num_feature_;
  return pa;
}

void Booster::run_predict(DMatrix* dm, PredictArgs pa, cudaStream_t s) {
  if (!dm->quantile) { launch_predict(pa, s); return; }
  if (pa.tree_end <= pa.tree_begin) return;
  // only the node slots of trees [tree_begin, tree_end) are mapped: an eval set maps each round's new trees once
  int64_t lo = h_tree_offset[pa.tree_begin], hi = h_tree_offset[pa.tree_begin + 1];
  for (int t = pa.tree_begin + 1; t < pa.tree_end; ++t) { lo = std::min(lo, h_tree_offset[t]); hi = std::max(hi, h_tree_offset[t + 1]); }
  bin_nodes_.ensure(std::max<size_t>(d_nodes.n, 1));     // indexed like d_nodes; grows (and is rewritten) with it
  launch_bin_thresholds(d_nodes.p + lo, (size_t)(hi - lo), dm->d_cut_ptrs.p, dm->d_cut_vals.p, dm->d_min_vals.p, dm->F, bin_nodes_.p + lo, s);
  pa.nodes = bin_nodes_.p;
  launch_predict_bins(pa, dm->binned_view(), s);
}

// the plan predict(dm, iteration_range = [iter_begin, iter_end)) executes (iter_end == 0: every round)
std::string Booster::debug_predict_plan(DMatrix* dm, int iter_begin, int iter_end) {
  configure();
  upload_model();
  if (iter_end == 0) iter_end = layers();
  B200_CHECK(iter_begin >= 0 && iter_begin <= iter_end && iter_end <= layers(), "debug_predict_plan: invalid iteration range");
  const PredictArgs pa = predict_args(dm, iteration_indptr_[iter_begin], iteration_indptr_[iter_end]);
  return predict_plan_json(dm->quantile ? plan_for_bins(pa, dm->binned_view()) : plan_for(pa), pa.tree_begin, pa.tree_end, pa.has_nan != 0);
}

// device time of the predictor kernel alone (margins of all trees into the scratch buffer), for the roofline line of bench.py
float Booster::debug_predict_kernel_ms(DMatrix* dm, int repeats) {
  configure();
  cudaStream_t s = engine_stream();
  upload_model();
  const int K = param_.num_outputs();
  pred_margin_.ensure((size_t)dm->n * K);
  PredictArgs pa = predict_args(dm, 0, (int)trees_.size());
  pa.margin = pred_margin_.p;
  cudaEvent_t e0, e1; CUDA_OK(cudaEventCreate(&e0)); CUDA_OK(cudaEventCreate(&e1));
  float total = 0.f;
  for (int r = 0; r < std::max(1, repeats); ++r) {
    launch_fill(pred_margin_.p, dm->n * K, base_margin(), s);
    CUDA_OK(cudaEventRecord(e0, s));
    run_predict(dm, pa, s);
    CUDA_OK(cudaEventRecord(e1, s));
    CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0; CUDA_OK(cudaEventElapsedTime(&ms, e0, e1)); total += ms;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return total / std::max(1, repeats);
}

void Booster::cached_margin(DMatrix* dm, std::vector<float>* out) {
  configure();
  cudaStream_t s = engine_stream();
  PredCache& c = cache_for(dm);
  bring_cache_up_to_date(dm, c);
  out->resize((size_t)dm->n * param_.num_outputs());
  if (!out->empty()) CUDA_OK(cudaMemcpyAsync(out->data(), c.margin.p, sizeof(float) * out->size(), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
}

void Booster::set_profile(bool on) { builder_->set_profile(on); }
std::string Booster::get_profile() { return builder_->profile_json(); }

}  // namespace b200
