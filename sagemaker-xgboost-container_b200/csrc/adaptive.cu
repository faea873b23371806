// adaptive.cu -- reg:absoluteerror and reg:quantileerror (adaptive.h): their gradient passes, the quantile metric, and the leaf
// refresh after each tree's structure is final: every leaf's value becomes fl(q * lr), q the alpha-quantile (0.5 for absolute
// error, the tree's target's quantile_alpha entry for quantile error) of the residuals of the leaf's rows [UPSTREAM-RECALL:
// src/objective/regression_obj.cu MeanAbsoluteError, src/objective/quantile_obj.cu, src/objective/adaptive.{h,cc,cu},
// src/common/stats.h].
// q is found by an exact radix select over order-preserving uint32 keys of the residuals, kSelectDigitBits per pass: each pass
// builds per-segment digit histograms of row counts and h_q (exact int64, all-reduced across ranks), and a pick kernel narrows
// each segment to one digit.  Nothing depends on row order, timing or the number of ranks (DESIGN.md §3).
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>
#include "adaptive.h"
#include "comm.h"
#include "rng.h"

namespace b200 {

static inline unsigned grid_for(int64_t n) { int64_t g = (n + 255) / 256; if (g < 1) g = 1; if (g > engine_num_sms() * 8) g = engine_num_sms() * 8; return (unsigned)g; }

// ---------------------------------------------------------------------------------------------
// gradient: g = sign(m - y) * w (sign(0) = 0), h = w [UPSTREAM-RECALL: MeanAbsoluteError::GetGradient]; r = fl(y - m)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) abserr_gradient_kernel(AbsErrGradArgs a) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float y = a.label[r], w = a.weight ? a.weight[r] : 1.0f, m = a.margin ? a.margin[r] : 0.f;
    const float diff = __fsub_rn(m, y);
    float g = __fmul_rn((float)((diff > 0.f) - (diff < 0.f)), w), h = w;
    if (a.subsample < 1.0f && !(rng_uniform(a.seed, 0x2000ull + a.iter, (unsigned long long)(r + a.row_offset)) < a.subsample)) { g = 0.f; h = 0.f; }
    if (a.resid) a.resid[r] = __fsub_rn(y, m);
    if (a.dense_g) reinterpret_cast<float*>(a.gpair)[r] = g; else a.gpair[r] = make_float2(g, h);
    mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  __shared__ float sg[8], sh[8];
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
  __syncthreads();
  if (threadIdx.x == 0 && a.absmax) {
    for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
    atomicMax(a.absmax, __float_as_uint(mg)); atomicMax(a.absmax + 1, __float_as_uint(mh));
  }
}
void launch_abserr_gradient(const AbsErrGradArgs& a, cudaStream_t s) {
  abserr_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// gradient of reg:quantileerror: per target j, d = m - y, g = (d >= 0 ? 1 - alpha_j : -alpha_j) * w, h = w; r = fl(y - m)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) quantile_gradient_kernel(QuantileGradArgs a) {
  __shared__ float sg[8], sh[8];
  for (int j = 0; j < a.Q; ++j) {          // target by target: each folds its own max|g| and max h
    const float alpha = a.alpha[j];
    float mg = 0.f, mh = 0.f;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
      const float y = a.label[r], w = a.weight ? a.weight[r] : 1.0f, m = a.margin ? a.margin[r * a.Q + j] : 0.f;
      const float diff = __fsub_rn(m, y);
      float g = diff >= 0.f ? __fmul_rn(__fsub_rn(1.0f, alpha), w) : __fmul_rn(-alpha, w), h = w;
      if (a.subsample < 1.0f && !(rng_uniform(a.seed, 0x2000ull + a.iter, (unsigned long long)(r + a.row_offset)) < a.subsample)) { g = 0.f; h = 0.f; }
      if (a.resid) a.resid[j * a.n + r] = __fsub_rn(y, m);
      if (a.dense_g) reinterpret_cast<float*>(a.gpair)[r] = g; else a.gpair[j * a.gp_stride + r] = make_float2(g, h);
      mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
    if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
    __syncthreads();
    if (threadIdx.x == 0 && a.absmax) {
      for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
      unsigned* am = a.absmax + (a.per_target ? 2 * j : 0);
      atomicMax(am, __float_as_uint(mg)); atomicMax(am + 1, __float_as_uint(mh));
    }
    __syncthreads();
  }
}
void launch_quantile_gradient(const QuantileGradArgs& a, cudaStream_t s) {
  B200_CHECK(!a.dense_g || a.Q == 1, "quantile gradient: the dense g layout holds one target");
  quantile_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

__global__ void __launch_bounds__(256) quantile_metric_kernel(const float* margin, const float* label, const float* weight, const float* alpha,
                                                              int Q, int64_t n, double* out) {
  double s = 0, ws = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const float y = label[r], w = weight ? weight[r] : 1.0f;
    for (int j = 0; j < Q; ++j) {
      const float d = __fsub_rn(y, margin[r * Q + j]), al = alpha[j];
      const float loss = d >= 0.f ? __fmul_rn(al, d) : __fmul_rn(__fsub_rn(al, 1.0f), d);
      s += (double)__fmul_rn(loss, w); ws += (double)w;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(out, s); atomicAdd(out + 1, ws); }
}
void launch_quantile_metric(const float* margin, const float* label, const float* weight, const float* alpha, int Q, int64_t n, double* out,
                            cudaStream_t s) {
  if (n == 0) return;
  quantile_metric_kernel<<<grid_for(n), 256, 0, s>>>(margin, label, weight, alpha, Q, n, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// keys: -0.0 is +0.0 and every NaN the positive quiet NaN (one value above +inf), then the usual order-preserving flip
// (negative floats reversed below the positive ones).  No key is 0xffffffff, so ~key != 0 marks a key in select_min_kernel.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned select_key(float v) {
  unsigned b = __float_as_uint(v);
  if (b == 0x80000000u) b = 0u;
  if (isnan(v)) b = 0x7fc00000u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Histograms with at most this many entries (both planes) are accumulated in shared memory per CTA, then flushed.
constexpr int kSelectSmemEntries = 4096;

// One pass: every selected row whose key matches its segment's prefix above the pass's digit adds 1 (and h_q) to its digit.
template <bool SMEM>
__global__ void __launch_bounds__(256) select_hist_kernel(SelectArgs a, const SelectSeg* st, unsigned long long* hist, int pass) {
  extern __shared__ unsigned long long sm[];
  const size_t E = (size_t)a.nseg * kSelectBuckets;
  unsigned long long* H = SMEM ? sm : hist;
  if (SMEM) { for (size_t e = threadIdx.x; e < 2 * E; e += blockDim.x) sm[e] = 0; __syncthreads(); }
  const int shift = 32 - kSelectDigitBits * (pass + 1);
  const unsigned hi_mask = pass == 0 ? 0u : ~0u << (shift + kSelectDigitBits);
  const float scale = a.h ? a.scales[1] : 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const int s = a.seg[r];
    if (s < 0) continue;
    const unsigned key = select_key(a.values[r]);
    if (pass > 0 && (st[s].mode == 0 || ((key ^ st[s].prefix) & hi_mask) != 0u)) continue;
    const size_t e = (size_t)s * kSelectBuckets + ((key >> shift) & (kSelectBuckets - 1));
    atomicAdd(H + e, 1ull);
    if (a.h) { const unsigned hq = (unsigned)__float2int_rn(a.h[r * a.h_stride] * scale); if (hq) atomicAdd(H + E + e, (unsigned long long)hq); }
  }
  if (SMEM) {
    __syncthreads();
    for (size_t e = threadIdx.x; e < 2 * E; e += blockDim.x) if (sm[e]) atomicAdd(hist + e, sm[e]);
  }
}

// After pass `pass`: each segment takes the digit holding its target and keeps the target's rank inside it.  Pass 0 first sets
// the target from the segment's totals, with upstream's rules: Quantile (x = alpha (n + 1), k = floor(x) - 1, d = x - 1 - k,
// ends clamped) for counts, WeightedQuantile (first cumulative weight >= alpha * total) for h_q.
__global__ void select_pick_kernel(SelectArgs a, SelectSeg* st, const unsigned long long* hist, int pass) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.nseg) return;
  const size_t E = (size_t)a.nseg * kSelectBuckets;
  const unsigned long long* hc = hist + (size_t)s * kSelectBuckets;
  const unsigned long long* hw = hc + E;
  SelectSeg g = st[s];
  if (pass == 0) {
    long long cnt = 0, wsum = 0;
    for (int b = 0; b < kSelectBuckets; ++b) { cnt += (long long)hc[b]; wsum += (long long)hw[b]; }
    g.prefix = 0u; g.need_v1 = 0; g.unused = 0; g.d = -1.0; g.target = 0; g.mode = cnt > 0 ? 1 : 0;
    if (cnt > 0 && a.h) {
      const double c = ceil(a.alpha * (double)wsum);
      if (wsum > 0 && c >= 1.0) { g.mode = 2; g.target = (long long)c; }     // else (every h_q rounds to 0, or alpha 0): the smallest key
    } else if (cnt > 0) {
      const double nd = (double)cnt;
      if (a.alpha <= 1.0 / (nd + 1.0)) g.target = 0;
      else if (a.alpha >= nd / (nd + 1.0)) g.target = cnt - 1;
      else { const double x = a.alpha * (nd + 1.0), k = floor(x) - 1.0; g.target = (long long)k; g.d = (x - 1.0) - k; }
    }
  }
  if (g.mode != 0) {
    const int shift = 32 - kSelectDigitBits * (pass + 1);
    const unsigned long long* hv = g.mode == 2 ? hw : hc;
    long long cum = 0; int b = 0;
    for (; b < kSelectBuckets - 1; ++b) {
      const long long v = (long long)hv[b];
      if (g.mode == 1 ? g.target < cum + v : g.target <= cum + v) break;
      cum += v;
    }
    g.target -= cum; g.prefix |= (unsigned)b << shift;
    if (pass == kSelectPasses - 1 && g.mode == 1 && g.d >= 0.0) g.need_v1 = g.target + 1 >= (long long)hc[b] ? 1 : 0;   // hc[b]: keys equal to v0
  }
  st[s] = g;
}

// The segments that need it: the smallest key above the selected one, as max(~key) (the all-reduce has max, not min).
template <bool SMEM>
__global__ void __launch_bounds__(256) select_min_kernel(SelectArgs a, const SelectSeg* st, unsigned* inv_min) {
  extern __shared__ unsigned smin[];
  unsigned* M = SMEM ? smin : inv_min;
  if (SMEM) { for (int e = threadIdx.x; e < a.nseg; e += blockDim.x) smin[e] = 0u; __syncthreads(); }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const int s = a.seg[r];
    if (s < 0 || !st[s].need_v1) continue;
    const unsigned key = select_key(a.values[r]);
    if (key > st[s].prefix) atomicMax(M + s, ~key);
  }
  if (SMEM) {
    __syncthreads();
    for (int e = threadIdx.x; e < a.nseg; e += blockDim.x) if (smin[e]) atomicMax(inv_min + e, smin[e]);
  }
}

// q = v0 + d (v1 - v0) in upstream's types: float difference, double product and sum, rounded to float once
__global__ void select_finish_kernel(SelectArgs a, const SelectSeg* st, const unsigned* inv_min, float* q) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.nseg) return;
  const SelectSeg g = st[s];
  float v = __int_as_float(0x7fc00000);
  if (g.mode != 0) {
    const float v0 = key_value(g.prefix);
    v = v0;
    if (g.mode == 1 && g.d >= 0.0) {
      const float v1 = g.need_v1 ? key_value(~inv_min[s]) : v0;
      v = __double2float_rn(__dadd_rn((double)v0, __dmul_rn(g.d, (double)__fsub_rn(v1, v0))));
    }
    if (a.split_cond) a.split_cond[a.leaf_nid[s]] = __fmul_rn(v, a.lr);
  }
  q[s] = v;
}

void segmented_select(const SelectArgs& a, SelectScratch* sc, const std::function<void(unsigned long long*, size_t)>& sum_i64,
                      const std::function<void(unsigned*, size_t)>& max_u32, cudaStream_t s) {
  B200_CHECK(a.nseg >= 1 && a.nseg <= sc->nseg, "segmented_select: more segments than the scratch holds");
  const size_t E = (size_t)a.nseg * kSelectBuckets;
  const bool smem = 2 * E <= (size_t)kSelectSmemEntries;
  const unsigned grid = grid_for(a.n), sgrid = (unsigned)((a.nseg + 255) / 256);
  for (int pass = 0; pass < kSelectPasses; ++pass) {
    CUDA_OK(cudaMemsetAsync(sc->hist.p, 0, 2 * E * sizeof(unsigned long long), s));
    if (smem) select_hist_kernel<true><<<grid, 256, 2 * E * sizeof(unsigned long long), s>>>(a, sc->st.p, sc->hist.p, pass);
    else select_hist_kernel<false><<<grid, 256, 0, s>>>(a, sc->st.p, sc->hist.p, pass);
    ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    sum_i64(sc->hist.p, 2 * E);
    select_pick_kernel<<<sgrid, 256, 0, s>>>(a, sc->st.p, sc->hist.p, pass); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  }
  CUDA_OK(cudaMemsetAsync(sc->inv_min.p, 0, sizeof(unsigned) * a.nseg, s));
  if (a.nseg <= kSelectSmemEntries) select_min_kernel<true><<<grid, 256, sizeof(unsigned) * a.nseg, s>>>(a, sc->st.p, sc->inv_min.p);
  else select_min_kernel<false><<<grid, 256, 0, s>>>(a, sc->st.p, sc->inv_min.p);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  max_u32(sc->inv_min.p, (size_t)a.nseg);
  select_finish_kernel<<<sgrid, 256, 0, s>>>(a, sc->st.p, sc->inv_min.p, sc->q.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

bool SelectScratch::ensure(int64_t n, int nseg_, int cap_nodes, int targets) {
  // every buffer a captured tree reads: a graph bakes in their addresses
  const void* before[9] = {hist.p, st.p, inv_min.p, q.p, leaf_nid.p, seg.p, resid.p, leaf_of_node.p, scales.p};
  hist.ensure((size_t)2 * nseg_ * kSelectBuckets); st.ensure(nseg_); inv_min.ensure(nseg_); q.ensure(nseg_); leaf_nid.ensure(nseg_);
  seg.ensure((size_t)std::max<int64_t>(n, 1)); resid.ensure((size_t)std::max<int64_t>(n, 1) * std::max(targets, 1)); leaf_of_node.ensure((size_t)std::max(cap_nodes, 1));
  absmax.ensure(2); scales.ensure(4);
  nseg = std::max(nseg, nseg_);
  const void* after[9] = {hist.p, st.p, inv_min.p, q.p, leaf_nid.p, seg.p, resid.p, leaf_of_node.p, scales.p};
  return memcmp(before, after, sizeof before) != 0;
}

// ---------------------------------------------------------------------------------------------
// training: dense leaf numbering (node order) and each row's leaf
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) number_leaves_kernel(TreeArrays t, const int* n_nodes, int* leaf_of_node, int* leaf_nid) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  const int nn = *n_nodes;
  int base = 0;
  for (int start = 0; start < nn; start += 1024) {
    const int i = start + threadIdx.x;
    const int leaf = i < nn && t.left[i] == -1 ? 1 : 0;
    int idx, total;
    Scan(tmp).ExclusiveSum(leaf, idx, total);
    if (i < nn) leaf_of_node[i] = leaf ? base + idx : -1;
    if (leaf) leaf_nid[base + idx] = i;
    base += total;
    __syncthreads();
  }
}
// the walk of update_margin_kernel (tree.cu) from the row's routed node or the root
__global__ void __launch_bounds__(256) locate_leaves_kernel(TreeArrays t, const uint8_t* bins_col, int64_t n, int has_missing, const uint8_t* node_of_row,
                                                            const float2* gpair, const int* leaf_of_node, int* seg) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    if (gpair && gpair[r].y == 0.f) { seg[r] = -1; continue; }
    int nid = node_of_row ? (int)node_of_row[r] : 0;
    while (t.left[nid] != -1) {
      const int b = bins_col[(int64_t)t.split_index[nid] * n + r];
      const bool left = (has_missing && b == kMissingBin) ? (t.default_left[nid] != 0) : (b <= t.split_bin[nid]);
      nid = left ? t.left[nid] : t.right[nid];
    }
    seg[r] = leaf_of_node[nid];
  }
}
void launch_locate_leaves(const TreeArrays& t, const int* n_nodes, const uint8_t* bins_col, int64_t n, int has_missing,
                          const uint8_t* node_of_row, const float2* gpair, SelectScratch* sc, cudaStream_t s) {
  number_leaves_kernel<<<1, 1024, 0, s>>>(t, n_nodes, sc->leaf_of_node.p, sc->leaf_nid.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  if (n == 0) return;
  locate_leaves_kernel<<<grid_for(n), 256, 0, s>>>(t, bins_col, n, has_missing, node_of_row, gpair, sc->leaf_of_node.p, sc->seg.p);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// the whole-matrix entry: segments and weights from the caller, the grid from the largest weight and the row count
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) quantile_prep_kernel(const int* segs, const float* w, int64_t n, int nseg, int* seg, unsigned* absmax, int* err) {
  float mw = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    int s = segs ? segs[r] : 0;
    if (s >= nseg) { *err = 1; s = -1; }
    if (w) { if (w[r] == 0.f) s = -1; mw = fmaxf(mw, w[r]); }
    if (seg) seg[r] = s < 0 ? -1 : s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, o));
  if ((threadIdx.x & 31) == 0 && mw > 0.f) atomicMax(absmax + 1, __float_as_uint(mw));
}
// scales[1] = sh exactly as tree.cu scales_kernel derives it from max h
__global__ void weight_scale_kernel(const unsigned* absmax, float* scales, int grad_bits) {
  const float mh = __uint_as_float(absmax[1]);
  int eh = 0;
  if (mh > 0.f && isfinite(mh)) frexpf(mh, &eh);
  scales[1] = ldexpf(1.0f, grad_bits + 1 - eh);
}

// sc->scales[1] from the all-reduced largest weight folded into sc->absmax[1]
static void weight_scale(int64_t global_n, SelectScratch* sc, cudaStream_t s) {
  if (Comm::get().distributed()) Comm::get().allreduce_max_u32(sc->absmax.p, 2, s);
  weight_scale_kernel<<<1, 1, 0, s>>>(sc->absmax.p, sc->scales.p, grad_bits_for(global_n)); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

void weight_grid(const float* weights, int64_t n, int64_t global_n, SelectScratch* sc, cudaStream_t s) {
  CUDA_OK(cudaMemsetAsync(sc->absmax.p, 0, 2 * sizeof(unsigned), s));
  if (n) { quantile_prep_kernel<<<grid_for(n), 256, 0, s>>>(nullptr, weights, n, 1, nullptr, sc->absmax.p, nullptr); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
  weight_scale(global_n, sc, s);
}

void segmented_quantile(const float* values, const int* segs, const float* weights, int64_t n, int64_t global_n, int nseg, double alpha,
                        float* out, SelectScratch* sc, cudaStream_t s) {
  B200_CHECK(nseg >= 1 && nseg <= (1 << 24), "segmented quantile: the segment count must be in [1, 2^24]");
  B200_CHECK(alpha >= 0.0 && alpha <= 1.0, "segmented quantile: alpha must be in [0, 1]");
  sc->ensure(n, nseg, 1);
  Comm& c = Comm::get();
  const bool dist = c.distributed();
  DevBuf<int> err; err.alloc(1); err.zero(s);
  CUDA_OK(cudaMemsetAsync(sc->absmax.p, 0, 2 * sizeof(unsigned), s));
  if (n) { quantile_prep_kernel<<<grid_for(n), 256, 0, s>>>(segs, weights, n, nseg, sc->seg.p, sc->absmax.p, err.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
  if (weights) weight_scale(global_n, sc, s);
  SelectArgs a{}; a.values = values; a.seg = sc->seg.p; a.h = weights; a.h_stride = 1; a.scales = sc->scales.p; a.n = n; a.nseg = nseg; a.alpha = alpha;
  segmented_select(a, sc, [&](unsigned long long* p, size_t cnt) { if (dist) c.allreduce_sum_i64(p, cnt, s); },
                   [&](unsigned* p, size_t cnt) { if (dist) c.allreduce_max_u32(p, cnt, s); }, s);
  int herr = 0;
  CUDA_OK(cudaMemcpyAsync(out, sc->q.p, sizeof(float) * nseg, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(&herr, err.p, sizeof herr, cudaMemcpyDeviceToHost, s));
  c.sync_stream(s);
  B200_CHECK(herr == 0, "segmented quantile: a segment id is not below the segment count");
}

}  // namespace b200
