// quantile.cu -- feature-quantile cut points on the device (SURVEY.md section 8a row A6).
// Upstream xgboost builds cuts with a weighted GK sketch (src/common/quantile.cc, hist_util.cc); that sketch is
// not restatable bit-exactly, so product and oracle share an EXACT definition instead (oracle/gbt_oracle.c
// cuts_from_distinct): sort each feature, collapse to distinct values with weights, then
//   m <= max_bin : cuts = distinct[1..m-1] U {last + (|last| + 1e-5)}          (identical to upstream)
//   m >  max_bin : cut k = the distinct value following the one whose cumulative weight reaches k*W/max_bin.
// One-time cost per DMatrix; uses CUB device primitives (sort / run-length / segmented sum), not on the per-round path.
#include <cub/cub.cuh>
#include <algorithm>
#include <climits>
#include <cmath>
#include "engine.h"
#include "misc.h"

namespace b200 {

__global__ void extract_col_kernel(const float* X, int64_t n, int F, int f, const float* w, float* keys, float* wout) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    float v = X[r * F + f];
    bool nan = isnan(v);
    keys[r] = nan ? __int_as_float(0x7f800000) : (v == 0.f ? 0.f : v);      // NaN -> +inf: sorts last; -0.0 -> +0.0 so that the
                                                                            // representative of the zero run (a cut value) does not depend on sort order / rank count
    if (wout) wout[r] = nan ? 0.f : (w ? w[r] : 1.f);
  }
}
__global__ void count_valid_kernel(const float* X, int64_t n, int F, int f, unsigned long long* out) {
  unsigned long long c = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) c += isnan(X[r * F + f]) ? 0ull : 1ull;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
struct ToDouble { __host__ __device__ double operator()(float x) const { return (double)x; } };

// Per feature: sort the column, run-length encode it, and take each distinct value's weight.  Weighted columns sum the
// weights of a run in double with one segmented reduction: one block per run, in an order fixed by the run's length, so
// the sums depend on the input alone (no float accumulation, no decoupled look-back).  The cumulative weights are then
// taken on the host, in value order.
void compute_summaries_device(const float* dX, int64_t n, int F, const float* dweights, int cap,
                              std::vector<FeatureSummary>* out, cudaStream_t s) {
  out->assign(F, FeatureSummary());
  if (n == 0) return;
  B200_CHECK(n <= (int64_t)INT_MAX, "quantile cuts: more than 2^31-1 rows on one GPU are not supported");
  const int ni = (int)n;
  DevBuf<float> keys, keys2, wts, wts2, uniq;
  DevBuf<int> counts, nruns, offs;
  DevBuf<double> wsum;
  DevBuf<unsigned long long> nvalid;
  keys.alloc(n); keys2.alloc(n); uniq.alloc(n); counts.alloc(n); nruns.alloc(1); nvalid.alloc(1);
  const bool weighted = dweights != nullptr;
  if (weighted) { wts.alloc(n); wts2.alloc(n); wsum.alloc(n); offs.alloc(n + 1); }
  cub::TransformInputIterator<double, ToDouble, const float*> wdouble(wts2.p, ToDouble());
  size_t tmp_bytes = 0, need = 0;
  // temp storage: max over the primitives used
  if (weighted) { cub::DeviceRadixSort::SortPairs(nullptr, need, keys.p, keys2.p, wts.p, wts2.p, (int64_t)n, 0, 32, s); tmp_bytes = std::max(tmp_bytes, need);
    cub::DeviceSegmentedReduce::Sum(nullptr, need, wdouble, wsum.p, ni, offs.p, offs.p + 1, s); tmp_bytes = std::max(tmp_bytes, need); }
  else { cub::DeviceRadixSort::SortKeys(nullptr, need, keys.p, keys2.p, (int64_t)n, 0, 32, s); tmp_bytes = std::max(tmp_bytes, need); }
  cub::DeviceRunLengthEncode::Encode(nullptr, need, keys2.p, uniq.p, counts.p, nruns.p, ni, s); tmp_bytes = std::max(tmp_bytes, need);
  DevBuf<unsigned char> tmp; tmp.alloc(tmp_bytes + 16);
  const int grid = (int)std::min<int64_t>((n + 255) / 256, engine_num_sms() * 16);
  std::vector<float> v; std::vector<int> cnt; std::vector<int> off; std::vector<double> w, c;
  for (int f = 0; f < F; ++f) {
    extract_col_kernel<<<grid, 256, 0, s>>>(dX, n, F, f, dweights, keys.p, weighted ? wts.p : nullptr); ++g_kernel_launches;
    CUDA_OK(cudaMemsetAsync(nvalid.p, 0, 8, s));
    count_valid_kernel<<<grid, 256, 0, s>>>(dX, n, F, f, nvalid.p); ++g_kernel_launches;
    size_t tb = tmp_bytes;
    if (weighted) CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys2.p, wts.p, wts2.p, (int64_t)n, 0, 32, s));
    else CUDA_OK(cub::DeviceRadixSort::SortKeys(tmp.p, tb, keys.p, keys2.p, (int64_t)n, 0, 32, s));
    tb = tmp_bytes;
    CUDA_OK(cub::DeviceRunLengthEncode::Encode(tmp.p, tb, keys2.p, uniq.p, counts.p, nruns.p, ni, s));
    int m = 0; unsigned long long nv = 0;
    CUDA_OK(cudaMemcpyAsync(&m, nruns.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaMemcpyAsync(&nv, nvalid.p, 8, cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    v.resize(m); cnt.resize(m);
    CUDA_OK(cudaMemcpyAsync(v.data(), uniq.p, sizeof(float) * m, cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaMemcpyAsync(cnt.data(), counts.p, sizeof(int) * m, cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    if (weighted && m > 0) {       // run i spans sorted rows [off[i], off[i + 1]); NaN rows carry weight 0
      off.resize(m + 1); off[0] = 0;
      for (int i = 0; i < m; ++i) off[i + 1] = off[i] + cnt[i];
      CUDA_OK(cudaMemcpyAsync(offs.p, off.data(), sizeof(int) * (m + 1), cudaMemcpyHostToDevice, s));
      tb = tmp_bytes;
      CUDA_OK(cub::DeviceSegmentedReduce::Sum(tmp.p, tb, wdouble, wsum.p, m, offs.p, offs.p + 1, s));
      w.resize(m);
      CUDA_OK(cudaMemcpyAsync(w.data(), wsum.p, sizeof(double) * m, cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaStreamSynchronize(s));
    }
    // Missing entries are keyed +inf, so they end the last run.  That run is dropped only when it holds nothing else: real
    // +inf values are a distinct value of their own.
    const int64_t nmiss = n - (int64_t)nv;
    if (nmiss > 0) { if (cnt[m - 1] == nmiss) m -= 1; else cnt[m - 1] -= (int)nmiss; }
    FeatureSummary& fs = (*out)[f];
    if (m <= 0) continue;
    if (!weighted) { w.resize(m); for (int i = 0; i < m; ++i) w[i] = (double)cnt[i]; }
    c.resize(m);                    // inclusive cumulative weights
    double acc = 0; for (int i = 0; i < m; ++i) { acc += w[i]; c[i] = acc; }
    if (m <= cap) {
      fs.vals.assign(v.begin(), v.begin() + m); fs.weights.assign(w.begin(), w.begin() + m);
      continue;
    }
    // cap-point summary plus the first distinct value (so the minimum survives): point k is the first distinct value whose
    // cumulative weight reaches W (k + 1) / cap; a point's weight is the difference of the cumulative weights
    const double W = c[m - 1];
    std::vector<int> idx(1, 0);
    for (int k = 0; k < cap; ++k) {
      const double target = W * (double)(k + 1) / (double)cap;
      const int i = (int)(std::lower_bound(c.begin(), c.begin() + (m - 1), target) - c.begin());
      if (v[i] > v[idx.back()]) idx.push_back(i);
    }
    for (size_t j = 0; j < idx.size(); ++j) {
      fs.vals.push_back(v[idx[j]]);
      fs.weights.push_back(c[idx[j]] - (j ? c[idx[j - 1]] : 0.0));
    }
  }
}

void merge_summaries(const std::vector<std::vector<FeatureSummary>>& per_rank, int F, std::vector<FeatureSummary>* merged) {
  merged->assign(F, FeatureSummary());
  for (int f = 0; f < F; ++f) {
    std::vector<std::pair<float, double>> pts;
    for (const auto& r : per_rank) for (size_t i = 0; i < r[f].vals.size(); ++i) pts.emplace_back(r[f].vals[i], r[f].weights[i]);
    std::stable_sort(pts.begin(), pts.end(), [](const std::pair<float, double>& a, const std::pair<float, double>& b) { return a.first < b.first; });
    FeatureSummary& out = (*merged)[f];
    for (auto& pw : pts) {
      if (!out.vals.empty() && out.vals.back() == pw.first) out.weights.back() += pw.second;
      else { out.vals.push_back(pw.first); out.weights.push_back(pw.second); }
    }
  }
}

void compute_rank_cuts_device(const float* dX, int F, const float* dweights, const int64_t* row_bounds, int nranges, int max_bin,
                              bool has_missing, HostCuts* out, cudaStream_t s) {
  std::vector<std::vector<FeatureSummary>> per_rank(nranges);
  for (int r = 0; r < nranges; ++r) {
    const int64_t b = row_bounds[r], e = row_bounds[r + 1];
    compute_summaries_device(dX + b * F, e - b, F, dweights ? dweights + b : nullptr, kRankSummaryCap, &per_rank[r], s);
  }
  std::vector<FeatureSummary> merged;
  merge_summaries(per_rank, F, &merged);
  cuts_from_summaries(merged, max_bin, has_missing, out);
}

// Same arithmetic as oracle/gbt_oracle.c cuts_from_distinct (shared definition, independently written here).
void cuts_from_summaries(const std::vector<FeatureSummary>& sums, int max_bin, bool has_missing, HostCuts* out) {
  int nb = std::min(max_bin, 256);
  if (has_missing && nb > 255) nb = 255;
  const int F = (int)sums.size();
  out->ptrs.assign(1, 0); out->vals.clear(); out->mins.assign(F, 0.f);
  for (int f = 0; f < F; ++f) {
    const std::vector<float>& d = sums[f].vals; const std::vector<double>& cw = sums[f].weights;
    const int64_t m = (int64_t)d.size();
    if (m == 0) { out->vals.push_back(1e-5f); out->mins[f] = -1e-5f; out->ptrs.push_back((int)out->vals.size()); continue; }
    if (m <= nb) { for (int64_t i = 1; i < m; ++i) out->vals.push_back(d[i]); }
    else {
      double W = 0; for (int64_t i = 0; i < m; ++i) W += cw[i];
      double cum = 0; int64_t i = 0; float last = d[0];
      for (int k = 1; k < nb; ++k) {
        double target = W * (double)k / (double)nb;
        while (i < m && cum + cw[i] < target) { cum += cw[i]; ++i; }
        int64_t j = i + 1 < m ? i + 1 : m - 1;
        float c = d[j];
        if (c > last) { out->vals.push_back(c); last = c; }
      }
    }
    float lastv = d[m - 1];
    out->vals.push_back(lastv + (std::fabs(lastv) + 1e-5f));
    out->mins[f] = d[0] - (std::fabs(d[0]) + 1e-5f);
    out->ptrs.push_back((int)out->vals.size());
  }
}

void compute_cuts_device(const float* dX, int64_t n, int F, const float* dweights, int max_bin, bool has_missing,
                         HostCuts* out, cudaStream_t s) {
  std::vector<FeatureSummary> sums;
  // single-rank path: exact (cap = everything). The distributed path merges capped summaries first (engine).
  compute_summaries_device(dX, n, F, dweights, (int)std::min<int64_t>(n > 0 ? n : 1, (int64_t)1 << 30), &sums, s);
  cuts_from_summaries(sums, max_bin, has_missing, out);
}

// ---------------------------------------------------------------------------------------------
// tree_method=approx: the cuts of every tree from its hessian (DESIGN.md "Approx")
// ---------------------------------------------------------------------------------------------
// Missing entries take the one positive quiet NaN, which the radix sort places after +inf: a column's first nv sorted entries
// are then exactly its values, +inf included.  -0.0 joins +0.0 as in extract_col_kernel.
__global__ void approx_keys_kernel(const float* X, int64_t n, int F, int f, float* keys, int* rows) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const float v = X[r * F + f];
    keys[r] = isnan(v) ? __int_as_float(0x7fc00000) : (v == 0.f ? 0.f : v);
    rows[r] = (int)r;
  }
}

__global__ void hessian_column_kernel(const float2* gp, int64_t n, float* out) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) out[r] = gp[r].y;
}
void launch_hessian_column(const float2* gp, int64_t n, float* out, cudaStream_t s) {
  if (n <= 0) return;
  hessian_column_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, engine_num_sms() * 16), 256, 0, s>>>(gp, n, out); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}

// grows d to hold `need` elements, keeping its first `used` (doubling, so a build copies each element O(1) times)
template <typename T> static void grow_keep(DevBuf<T>& d, size_t used, size_t need, cudaStream_t s) {
  if (need <= d.n) return;
  DevBuf<T> bigger; bigger.alloc(std::max(need, 2 * d.n));
  if (used) CUDA_OK(cudaMemcpyAsync(bigger.p, d.p, sizeof(T) * used, cudaMemcpyDeviceToDevice, s));
  std::swap(bigger.p, d.p); std::swap(bigger.n, d.n);
}

void approx_sketch_build(const float* dX, int64_t n, int F, int nb, const HostCuts& cuts, ApproxSketch* sk, cudaStream_t s) {
  B200_CHECK(n <= (int64_t)INT_MAX, "tree_method=approx: more than 2^31-1 rows on one GPU are not supported");
  const int ni = (int)n;
  sk->F = F; sk->nb = nb; sk->n = n;
  DevBuf<float> keys, keys2, uniq; DevBuf<int> rows, counts, nruns; DevBuf<unsigned long long> nvalid;
  const size_t n1 = (size_t)std::max<int64_t>(n, 1);
  keys.alloc(n1); keys2.alloc(n1); uniq.alloc(n1); rows.alloc(n1); counts.alloc(n1); nruns.alloc(1); nvalid.alloc(1);
  // a kept feature's order is sorted straight to the end of sk->order, its run starts scanned straight to the end of
  // sk->run_start; a feature that turns out not to be kept is simply not counted
  sk->order.alloc(n1); sk->run_start.alloc(n1);
  size_t tmp_bytes = 0, need = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, need, keys.p, keys2.p, rows.p, sk->order.p, ni, 0, 32, s); tmp_bytes = std::max(tmp_bytes, need);
  cub::DeviceRunLengthEncode::Encode(nullptr, need, keys2.p, uniq.p, counts.p, nruns.p, ni, s); tmp_bytes = std::max(tmp_bytes, need);
  cub::DeviceScan::ExclusiveSum(nullptr, need, counts.p, sk->run_start.p, ni, s); tmp_bytes = std::max(tmp_bytes, need);
  DevBuf<unsigned char> tmp; tmp.alloc(tmp_bytes + 16);
  const int grid = (int)std::min<int64_t>((n + 255) / 256 + 1, engine_num_sms() * 16);
  // One sort per feature, kept for the features with more distinct values than bins: the cuts of the others are their distinct
  // values whatever the weights, so they stay as the matrix has them.
  std::vector<int64_t> elem_off{0}, run_off{0};
  std::vector<int> active;
  for (int f = 0; f < F && n > 0; ++f) {
    const int64_t e0 = elem_off.back(), r0 = run_off.back();
    grow_keep(sk->order, (size_t)e0, (size_t)e0 + n1, s);
    approx_keys_kernel<<<grid, 256, 0, s>>>(dX, n, F, f, keys.p, rows.p); ++g_kernel_launches;
    CUDA_OK(cudaMemsetAsync(nvalid.p, 0, 8, s));
    count_valid_kernel<<<grid, 256, 0, s>>>(dX, n, F, f, nvalid.p); ++g_kernel_launches;
    size_t tb = tmp_bytes;
    CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys2.p, rows.p, sk->order.p + e0, ni, 0, 32, s));
    unsigned long long nv = 0;
    CUDA_OK(cudaMemcpyAsync(&nv, nvalid.p, 8, cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    int m = 0;
    if (nv > 0) {
      tb = tmp_bytes;
      CUDA_OK(cub::DeviceRunLengthEncode::Encode(tmp.p, tb, keys2.p, uniq.p, counts.p, nruns.p, (int)nv, s));
      CUDA_OK(cudaMemcpyAsync(&m, nruns.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaStreamSynchronize(s));
    }
    if (m <= nb) continue;
    grow_keep(sk->run_start, (size_t)r0, (size_t)r0 + m, s);
    tb = tmp_bytes;
    CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp.p, tb, counts.p, sk->run_start.p + r0, m, s));      // integer: exact in any order
    active.push_back(f);
    elem_off.push_back(e0 + (int64_t)nv); run_off.push_back(r0 + m);
  }
  sk->A = (int)active.size(); sk->nruns = run_off.back();
  auto fit = [&](auto& d, size_t used) {         // the kept entries only, not the doubling's slack
    std::remove_reference_t<decltype(d)> exact; exact.alloc(std::max<size_t>(used, 1));
    if (used) CUDA_OK(cudaMemcpyAsync(exact.p, d.p, sizeof(*d.p) * used, cudaMemcpyDeviceToDevice, s));
    std::swap(exact.p, d.p); std::swap(exact.n, d.n);
    CUDA_OK(cudaStreamSynchronize(s));
  };
  fit(sk->order, (size_t)elem_off.back()); fit(sk->run_start, (size_t)sk->nruns);
  auto up = [&](auto& d, const auto& h) { d.alloc(std::max<size_t>(h.size(), 1));
    if (!h.empty()) CUDA_OK(cudaMemcpyAsync(d.p, h.data(), sizeof(h[0]) * h.size(), cudaMemcpyHostToDevice, s)); };
  up(sk->elem_off, elem_off); up(sk->run_off, run_off); up(sk->feat, active);
  sk->run_w.alloc(std::max<int64_t>(sk->nruns, 1));
  // the per-tree staging [F][256] holds the fixed cuts of the other features from the start
  std::vector<float> stage((size_t)F * kBins, 0.f); std::vector<int> scnt(F, 0);
  for (int f = 0; f < F; ++f) {
    scnt[f] = cuts.ptrs[f + 1] - cuts.ptrs[f];
    std::copy(cuts.vals.begin() + cuts.ptrs[f], cuts.vals.begin() + cuts.ptrs[f + 1], stage.begin() + (size_t)f * kBins);
  }
  up(sk->stage_vals, stage); up(sk->stage_cnt, scnt);
  CUDA_OK(cudaStreamSynchronize(s));                 // the host vectors and the temporaries die with this scope
  sk->valid = true;
}

// Each run's weight, in double, in an order fixed by the run alone: a warp takes 32 consecutive runs; a lane sums a run of at
// most 32 entries itself, in order, and the warp sums each longer run together (lane l takes its entries l, l + 32, ..., then a
// fixed butterfly).  The sums depend on the input alone, not on the grid or the SM count.  Continuous features are mostly
// single-entry runs, so the lanes stay busy.
constexpr int kShortRun = 32;
__global__ void approx_run_sum_kernel(const int* order, const int* run_start, const int64_t* elem_off, const int64_t* run_off, int A,
                                      int64_t nruns, const float2* gp, double* run_w) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; base < nruns; base += nw * 32) {
    const int64_t r = base + lane;
    int64_t b = 0, e = 0;
    if (r < nruns) {
      int lo = 0, hi = A;                      // the feature of run r: run_off[a] <= r < run_off[a + 1]
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (run_off[mid] <= r) lo = mid; else hi = mid; }
      const int64_t eb = elem_off[lo];
      b = eb + run_start[r]; e = r + 1 < run_off[lo + 1] ? eb + run_start[r + 1] : elem_off[lo + 1];
    }
    const bool is_long = e - b > kShortRun;
    if (r < nruns && !is_long) {
      double acc = 0.0;
      for (int64_t i = b; i < e; ++i) acc += (double)gp[order[i]].y;
      run_w[r] = acc;
    }
    for (unsigned longs = __ballot_sync(0xffffffffu, is_long); longs; longs &= longs - 1) {
      const int l = __ffs(longs) - 1;
      const int64_t lb = __shfl_sync(0xffffffffu, b, l), le = __shfl_sync(0xffffffffu, e, l);
      double acc = 0.0;
      for (int64_t i = lb + lane; i < le; i += 32) acc += (double)gp[order[i]].y;
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) run_w[base + l] = acc;
    }
  }
}

// Per feature (one block each): the inclusive cumulative weights of its runs, in place, by a block scan over chunks in order.
constexpr int kApproxThreads = 256, kApproxItems = 8;
__global__ void __launch_bounds__(kApproxThreads) approx_scan_kernel(const int64_t* run_off, double* run_w) {
  typedef cub::BlockScan<double, kApproxThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ double carry;
  const int64_t b = run_off[blockIdx.x], e = run_off[blockIdx.x + 1];
  if (threadIdx.x == 0) carry = 0.0;
  __syncthreads();
  for (int64_t c0 = b; c0 < e; c0 += kApproxThreads * kApproxItems) {
    double v[kApproxItems];
    for (int i = 0; i < kApproxItems; ++i) { const int64_t at = c0 + threadIdx.x * kApproxItems + i; v[i] = at < e ? run_w[at] : 0.0; }
    double total;
    Scan(tmp).InclusiveSum(v, v, total);
    const double c = carry;
    for (int i = 0; i < kApproxItems; ++i) { const int64_t at = c0 + threadIdx.x * kApproxItems + i; if (at < e) run_w[at] = c + v[i]; }
    __syncthreads();
    if (threadIdx.x == 0) carry = c + total;
    __syncthreads();
  }
}

// Per feature (one block each): the shared cut rule (cuts_from_summaries) on its runs.  Cut k (1 <= k < nb) is the value after
// the first run whose cumulative weight reaches W k / nb, kept when larger than the cut before it; the end cut follows.  A
// feature of weight 0 takes every target at run 0, so its cuts are its second distinct value and the end cut.
__global__ void __launch_bounds__(kApproxThreads) approx_select_kernel(const float* X, int F, const int* order, const int* run_start,
                                                                        const int64_t* elem_off, const int64_t* run_off, const int* feat,
                                                                        const double* cum, int nb, float* stage_vals, int* stage_cnt) {
  __shared__ float cand[kBins];
  const int a = blockIdx.x, f = feat[a];
  const int64_t r0 = run_off[a]; const int m = (int)(run_off[a + 1] - r0);
  const double* c = cum + r0;
  const double W = c[m - 1];
  auto value = [&](int j) { return X[(int64_t)order[elem_off[a] + run_start[r0 + j]] * F + f]; };
  for (int k = 1 + threadIdx.x; k < nb; k += blockDim.x) {
    const double target = W * (double)k / (double)nb;
    int lo = 0, hi = m;                        // first run with c >= target (m: none)
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (c[mid] < target) lo = mid + 1; else hi = mid; }
    cand[k] = value(lo + 1 < m ? lo + 1 : m - 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float* out = stage_vals + (size_t)f * kBins;
    float v = value(0);
    const float last = value(m - 1);
    const float x0 = v == 0.f ? 0.f : v;       // the key of -0.0 is +0.0
    float prev = x0; int cnt = 0;
    for (int k = 1; k < nb; ++k) { float x = cand[k]; x = x == 0.f ? 0.f : x; if (x > prev) { out[cnt++] = x; prev = x; } }
    const float l = last == 0.f ? 0.f : last;
    out[cnt++] = __fadd_rn(l, __fadd_rn(fabsf(l), 1e-5f));
    stage_cnt[f] = cnt;
  }
}

// cut_ptrs from the staged counts (one block, in chunks), then every feature's staged cuts to their place
__global__ void __launch_bounds__(1024) approx_ptrs_kernel(const int* stage_cnt, int F, int* cut_ptrs) {
  typedef cub::BlockScan<int, 1024> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  if (threadIdx.x == 0) { carry = 0; cut_ptrs[0] = 0; }
  __syncthreads();
  for (int c0 = 0; c0 < F; c0 += 1024) {
    const int f = c0 + threadIdx.x;
    int v = f < F ? stage_cnt[f] : 0, total;
    Scan(tmp).InclusiveSum(v, v, total);
    if (f < F) cut_ptrs[f + 1] = carry + v;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
}
__global__ void approx_place_kernel(const float* stage_vals, const int* cut_ptrs, int F, float* cut_vals) {
  for (int f = blockIdx.x; f < F; f += gridDim.x) {
    const int b = cut_ptrs[f], cnt = cut_ptrs[f + 1] - b;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) cut_vals[b + i] = stage_vals[(size_t)f * kBins + i];
  }
}

void approx_sketch_cuts(const float* dX, const ApproxSketch& sk, const float2* gp, int* cut_ptrs, float* cut_vals, cudaStream_t s) {
  if (sk.A > 0) {
    const int64_t warps = std::min<int64_t>((sk.nruns + 31) / 32, (int64_t)engine_num_sms() * 64);
    approx_run_sum_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, s>>>(sk.order.p, sk.run_start.p, sk.elem_off.p, sk.run_off.p, sk.A, sk.nruns, gp, sk.run_w.p);
    ++g_kernel_launches;
    approx_scan_kernel<<<sk.A, kApproxThreads, 0, s>>>(sk.run_off.p, sk.run_w.p); ++g_kernel_launches;
    approx_select_kernel<<<sk.A, kApproxThreads, 0, s>>>(dX, sk.F, sk.order.p, sk.run_start.p, sk.elem_off.p, sk.run_off.p, sk.feat.p, sk.run_w.p, sk.nb,
                                                         sk.stage_vals.p, sk.stage_cnt.p); ++g_kernel_launches;
  }
  approx_ptrs_kernel<<<1, 1024, 0, s>>>(sk.stage_cnt.p, sk.F, cut_ptrs); ++g_kernel_launches;
  approx_place_kernel<<<(unsigned)std::min(sk.F, engine_num_sms() * 8), 256, 0, s>>>(sk.stage_vals.p, cut_ptrs, sk.F, cut_vals); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}

}  // namespace b200
