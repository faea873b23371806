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

}  // namespace b200
