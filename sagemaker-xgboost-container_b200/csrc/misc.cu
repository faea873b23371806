// misc.cu -- objective gradients, feature binning, tree-traversal predictor and evaluation metrics.
// SURVEY.md section 8a rows A5, A5b, A6 (binning half), A11, A12.  Formulas restate upstream xgboost
// (src/objective/regression_loss.h, multiclass_obj.cu, src/data/gradient_index.cc, src/predictor/cpu_predictor.cc,
// src/metric/elementwise_metric.cu, multiclass_metric.cu) as written down in oracle/gbt_oracle.c.
#include <algorithm>
#include <cstdlib>
#include <utility>
#include "curve.h"
#include "elementwise.h"
#include "engine.h"
#include "inplace.h"
#include "misc.h"
#include "predict_tile.h"
#include "rng.h"
#include "transform.h"
#include "traverse.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// gradient pairs: one thread per row, all K classes; also the running max|g|, max h of the round.  With dense_g only g is
// stored (4 B per row instead of 8); h == 1.0f is still folded into max h, so the fixed-point scales keep their bits.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gradient_kernel(GradArgs a) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float y = a.label[r];
    float w = a.weight ? a.weight[r] : 1.0f;
    const bool dropped = !row_sampled(a.seed, a.iter, (unsigned long long)(r + a.row_offset), a.subsample);
    if (a.objective == kSoftprob || a.objective == kSoftmax) {
      const int K = a.K;
      const float* m = a.margin ? a.margin + r * K : nullptr;
      float wmax = m ? m[0] : 0.f;
      for (int k = 1; k < K; ++k) wmax = fmaxf(wmax, m ? m[k] : 0.f);
      float wsum = 0.f;
      for (int k = 0; k < K; ++k) wsum += expf((m ? m[k] : 0.f) - wmax);
      int label = (int)y;
      if (label < 0 || label >= K) { *a.err = 2; label = 0; }
      for (int k = 0; k < K; ++k) {
        float pk = expf((m ? m[k] : 0.f) - wmax) / wsum;
        float h = fmaxf(2.0f * pk * (1.0f - pk) * w, 1e-16f);
        float g = (label == k ? pk - 1.0f : pk) * w;
        if (dropped) { g = 0.f; h = 0.f; }
        a.gpair[(int64_t)k * a.gp_stride + r] = make_float2(g, h);
        mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
      }
    } else {
      if (objective_is_reg_loss(a.objective) && y == 1.0f) w *= a.scale_pos_weight;
      float g, h;
      elementwise_gradient(a.objective, y, a.margin ? a.margin[r] : 0.f, a.aux, a.err, &g, &h);
      g *= w; h *= w;
      if (dropped) { g = 0.f; h = 0.f; }
      if (a.dense_g) reinterpret_cast<float*>(a.gpair)[r] = g; else a.gpair[r] = make_float2(g, h);
      mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  __shared__ float sg[8], sh[8];
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
    if (a.absmax) { atomicMax(a.absmax, __float_as_uint(mg)); atomicMax(a.absmax + 1, __float_as_uint(mh)); }
  }
}

// one tree's row sample of a forest round: the kept rows' pairs of every class copied, the others zeroed, and max|g|, max h of
// the copy folded into absmax (the tree's fixed-point scales).  Reads and writes 8 K bytes per row.
__global__ void __launch_bounds__(256) sample_gpair_kernel(SampleArgs a) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const bool keep = rng_uniform(a.seed, a.stream, (unsigned long long)(r + a.row_offset)) < a.subsample;
    for (int k = 0; k < a.K; ++k) {
      const float2 v = keep ? a.src[(int64_t)k * a.gp_stride + r] : make_float2(0.f, 0.f);
      a.dst[(int64_t)k * a.gp_stride + r] = v;
      mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, v.y);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  __shared__ float sg[8], sh[8];
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
    atomicMax(a.absmax, __float_as_uint(mg)); atomicMax(a.absmax + 1, __float_as_uint(mh));
  }
}

// sum of (g,h) over rows in double (base-score stump)
__global__ void __launch_bounds__(256) sum_gpair_kernel(const float2* gp, int64_t n, double* out) {
  double g = 0, h = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) { float2 v = gp[r]; g += v.x; h += v.y; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { g += __shfl_xor_sync(0xffffffffu, g, o); h += __shfl_xor_sync(0xffffffffu, h, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(out, g); atomicAdd(out + 1, h); }
}

// ---------------------------------------------------------------------------------------------
// binning: float matrix (row-major, NaN = missing) -> uint8 codes in the layout of engine.h BinnedMatrix:
// main [n][ngroups*32] (byte column c == feature c) and tail [n][tw] (tail slot s == feature ngroups*32 + s)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t bin_of(float v, const float* c, int nc) {
  if (isnan(v)) return (uint8_t)kMissingBin;
  int lo = 0, hi = nc;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (c[mid] > v) hi = mid; else lo = mid + 1; }
  if (lo >= nc) lo = nc - 1;
  return (uint8_t)lo;
}

__global__ void __launch_bounds__(256) bin_kernel(const float* X, int64_t n, int F, int ngroups, int tw, const int* cut_ptrs, const float* cut_vals,
                                                  uint8_t* bins, uint8_t* bins_tail) {
  const int W = ngroups * kSlots + tw;                  // byte columns per row over both blocks
  const int64_t total = n * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % W);
    const int64_t r = idx / W;
    uint8_t b = 0;
    if (c < F) b = bin_of(X[r * F + c], cut_vals + cut_ptrs[c], cut_ptrs[c + 1] - cut_ptrs[c]);     // byte column == feature index in both blocks
    if (c < ngroups * kSlots) bins[r * (ngroups * kSlots) + c] = b;
    else bins_tail[r * tw + (c - ngroups * kSlots)] = b;
  }
}

// rows re-laid at `dst_stride` bytes (whole 128 B lines for 96 B rows): 16 B per thread.  The row's tw tail bytes go right
// behind its main bytes (offset src_stride), the rest of the pad is zero.
__global__ void __launch_bounds__(256) pad_rows_kernel(const uint8_t* src, const uint8_t* tail, int tw, int64_t n, int src_stride, uint8_t* dst, int dst_stride) {
  const int cpr = dst_stride / 16, spr = src_stride / 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * cpr; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cpr; const int c = (int)(i - r * cpr);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (c < spr) v = reinterpret_cast<const uint4*>(src + r * src_stride)[c];
    else if (c == spr && tw > 0) {
      v.x = reinterpret_cast<const unsigned*>(tail + r * tw)[0];
      if (tw == 8) v.y = reinterpret_cast<const unsigned*>(tail + r * tw)[1];
    }
    reinterpret_cast<uint4*>(dst + r * dst_stride)[c] = v;
  }
}
void launch_pad_rows(const uint8_t* src, const uint8_t* tail, int tw, int64_t n, int src_stride, uint8_t* dst, int dst_stride, cudaStream_t s) {
  if (n == 0) return;
  B200_CHECK(tw == 0 || (tw <= dst_stride - src_stride && src_stride % 16 == 0), "pad_rows: the tail does not fit in the row's pad");
  pad_rows_kernel<<<engine_num_sms() * 16, 256, 0, s>>>(src, tail, tw, n, src_stride, dst, dst_stride); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// column-major copy [F][n] of the binned matrix (used by the 1-byte-per-row consumers: partition, cache update)
__global__ void __launch_bounds__(256) transpose_bins_kernel(const uint8_t* bins, const uint8_t* bins_tail, int64_t n, int F, int ngroups, int tw, uint8_t* bins_col) {
  __shared__ uint8_t tile[256][kSlots + 1];
  const int g = blockIdx.y;                             // ngroups == the tail block
  const bool is_tail = g == ngroups;
  const int width = is_tail ? tw : kSlots;
  const int64_t r0 = (int64_t)blockIdx.x * 256;
  for (int i = threadIdx.x; i < 256 * width; i += 256) {
    int rr = i / width, s = i % width;
    int64_t r = r0 + rr;
    tile[rr][s] = r < n ? (is_tail ? bins_tail[r * tw + s] : bins[r * (ngroups * kSlots) + g * kSlots + s]) : 0;
  }
  __syncthreads();
  const int64_t r = r0 + threadIdx.x;
  if (r < n) for (int s = 0; s < width; ++s) { int f = g * kSlots + s; if (f < F) bins_col[(int64_t)f * n + r] = tile[threadIdx.x][s]; }
}

__global__ void __launch_bounds__(256) count_nan_kernel(const float* X, int64_t count, float missing, int use_missing, unsigned long long* out) {
  unsigned long long c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
    float v = X[i];
    c += (isnan(v) || (use_missing && v == missing)) ? 1ull : 0ull;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

__global__ void __launch_bounds__(256) replace_missing_kernel(float* X, int64_t count, float missing) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    if (X[i] == missing) X[i] = __int_as_float(0x7fc00000);
}

// ---------------------------------------------------------------------------------------------
// predictor: one thread per row, trees in model order, fp32 accumulation
// ---------------------------------------------------------------------------------------------
template <class Src>
__global__ void __launch_bounds__(256) predict_kernel(PredictArgs a, Src src) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n) return;
  const int nt = a.tree_end - a.tree_begin;
  float acc = (a.K == 1 && a.margin) ? a.margin[r] : 0.f;
  for (int t = a.tree_begin; t < a.tree_end; ++t) {
    DevNode nd;
    const int nid = tree_leaf_by(a.nodes + a.tree_offset[t], [&](unsigned f) { return src.at(r, (int)f); }, &nd);
    if (a.margin) { if (a.K == 1) acc += nd.cond; else a.margin[r * a.K + a.tree_info[t]] += nd.cond; }
    if (a.leaf) a.leaf[r * nt + (t - a.tree_begin)] = nid;
  }
  if (a.K == 1 && a.margin) a.margin[r] = acc;
}

// Block-cooperative predictor (BASELINE config 5): a CTA stages a tile of rows into shared memory with coalesced loads
// (the thread-per-row kernel above gathers 4 B at a time from a 4*F-byte row: 1 % of HBM peak in round 1) and keeps the
// trees there too, 8 B per node, so a traversal step is two LDS.  With T trees of depth D a row costs ~8*T*D instructions
// against 4*F bytes: beyond T*D ~ 100 the kernel is issue-bound, not HBM-bound (DESIGN.md "predictor").
// Src (inplace.h) stages a tile of rows: the DMatrix's float32 matrix, or an in-place input read at its own dtype and strides.
template <bool HAS_NAN, bool LEAF_OUT, class Src>
__global__ void __launch_bounds__(1024) predict_tiled_kernel(PredictArgs a, Src src, int tree_lo, int tree_hi, int pitch, int rows_per_tile, int64_t num_tiles) {
  extern __shared__ __align__(16) unsigned char psm[];
  int* s_toff; PNode* s_nodes;
  float* s_x = reinterpret_cast<float*>(stage_tree_chunk(a, tree_lo, tree_hi, psm, &s_toff, &s_nodes));
  const int nt_chunk = tree_hi - tree_lo;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t r0 = tile * rows_per_tile;
    const int rows = (int)((a.n - r0 < rows_per_tile) ? a.n - r0 : rows_per_tile);
    __syncthreads();                                                            // trees staged / previous tile consumed
    src.stage(s_x, pitch, r0, rows);
    __syncthreads();
    for (int rl = threadIdx.x; rl < rows; rl += blockDim.x) {
      const float* x = s_x + rl * pitch;
      predict_staged_row<LEAF_OUT>(a, s_nodes, s_toff, nt_chunk, tree_lo, r0 + rl, [&](const PNode& nd) {
        const float v = x[(nd.w >> 16) & 0x7fffu];
        bool go_left = v < nd.cond;
        if (HAS_NAN) { if (isnan(v)) go_left = (nd.w >> 31) != 0; }
        return go_left;
      });
    }
  }
}

// margins -> predictions (PredTransform), in place
__global__ void __launch_bounds__(256) transform_kernel(float* m, int64_t n, int K, int objective, float* out_class) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (objective == kSoftprob || objective == kSoftmax) {
    float* p = m + r * K;
    if (objective == kSoftmax) { out_class[r] = (float)softmax_class(p, K); return; }
    float wmax; const float wsum = softmax_sum(p, K, &wmax);
    for (int k = 0; k < K; ++k) p[k] = expf(p[k] - wmax) / wsum;
  } else m[r] = transform_one(m[r], objective);
}

// the scores of the curve metrics (curve.h): computed here, with this file's flags, so they are predict()'s values bit for bit
__global__ void __launch_bounds__(256) curve_scores_kernel(const float* margin, int64_t n, int K, int c, int logistic, float* key, int* iota) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    float p;
    if (K) { const float* m = margin + r * K; float wmax; const float wsum = softmax_sum(m, K, &wmax); p = expf(m[c] - wmax) / wsum; }
    else { p = margin[r]; if (logistic) p = sigmoidf_xgb(p); }
    key[r] = p == 0.0f ? 0.0f : p;        // -0.0 sorts as +0.0: one tie block
    iota[r] = (int)r;
  }
}

__global__ void __launch_bounds__(256) fill_kernel(float* p, int64_t n, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void __launch_bounds__(256) add_base_margin_kernel(float* p, const float* bm, int64_t count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) p[i] = bm[i];
}

// ---------------------------------------------------------------------------------------------
// element-wise evaluation metrics on raw margins: out[0] += sum(w * loss), out[1] += sum(w)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) metric_kernel(MetricArgs a) {
  double s = 0, ws = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float y = a.label[r];
    const float w = a.weight ? a.weight[r] : 1.0f;
    float loss = 0.f;
    if (a.metric == kMetricMlogloss || a.metric == kMetricMerror) {
      const float* m = a.margin + r * a.K;
      float wmax = m[0]; int arg = 0;
      for (int k = 1; k < a.K; ++k) if (m[k] > wmax) { wmax = m[k]; arg = k; }
      int label = (int)y;
      if (a.metric == kMetricMerror) loss = (arg != label) ? 1.f : 0.f;
      else {
        float wsum = 0.f;
        for (int k = 0; k < a.K; ++k) wsum += expf(m[k] - wmax);
        float p = (label >= 0 && label < a.K) ? expf(m[label] - wmax) / wsum : 0.f;
        const float eps = 1e-16f;
        loss = p > eps ? -logf(p) : -logf(eps);
      }
    } else {
      loss = elementwise_loss(a.metric, y, metric_prediction(a.margin[r], a.is_logistic, a.transform), a.threshold, a.aux);
    }
    s += (double)(loss * w); ws += (double)w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(a.out, s); atomicAdd(a.out + 1, ws); }
}

// ---------------------------------------------------------------------------------------------
static inline int grid_for(int64_t n, int block = 256, int cap = engine_num_sms() * 16) {
  int64_t g = (n + block - 1) / block; if (g < 1) g = 1; if (g > cap) g = cap; return (int)g;
}
void launch_gradient(const GradArgs& a, cudaStream_t s) {
  B200_CHECK(!a.dense_g || (a.K == 1 && a.objective == kSquaredError && a.weight == nullptr && a.subsample >= 1.0f),
             "gradient: the dense g layout is for constant-hessian objectives only");
  if (a.n == 0) return;
  gradient_kernel<<<grid_for(a.n, 256, engine_num_sms() * 8), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_sample_gpair(const SampleArgs& a, cudaStream_t s) {
  if (a.n == 0) return;
  sample_gpair_kernel<<<grid_for(a.n, 256, engine_num_sms() * 8), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_sum_gpair(const float2* gp, int64_t n, double* out, cudaStream_t s) {
  sum_gpair_kernel<<<grid_for(n), 256, 0, s>>>(gp, n, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_bin(const float* X, int64_t n, int F, int ngroups, int tw, const int* cut_ptrs, const float* cut_vals, uint8_t* bins, uint8_t* bins_tail, cudaStream_t s) {
  if (n == 0) return;
  bin_kernel<<<grid_for(n * (ngroups * kSlots + tw), 256, engine_num_sms() * 32), 256, 0, s>>>(X, n, F, ngroups, tw, cut_ptrs, cut_vals, bins, bins_tail); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}
void launch_transpose_bins(const uint8_t* bins, const uint8_t* bins_tail, int64_t n, int F, int ngroups, int tw, uint8_t* bins_col, cudaStream_t s) {
  if (n == 0) return;
  dim3 grid((unsigned)((n + 255) / 256), ngroups + (tw > 0 ? 1 : 0));
  transpose_bins_kernel<<<grid, 256, 0, s>>>(bins, bins_tail, n, F, ngroups, tw, bins_col); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_count_nan(const float* X, int64_t count, float missing, int use_missing, unsigned long long* out, cudaStream_t s) {
  if (count == 0) return;
  count_nan_kernel<<<grid_for(count), 256, 0, s>>>(X, count, missing, use_missing, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_replace_missing(float* X, int64_t count, float missing, cudaStream_t s) {
  if (count == 0) return;
  replace_missing_kernel<<<grid_for(count), 256, 0, s>>>(X, count, missing); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
// the plan (predict_plan.h) of these arguments: B200XGB_PREDICT_LEGACY (read once per process) forces thread-per-row
PredictPlan plan_for(const PredictArgs& a) {
  static const bool legacy = getenv("B200XGB_PREDICT_LEGACY") != nullptr;
  return plan_predict(a.h_tree_offset, a.tree_begin, a.tree_end, a.F, a.model_F, a.children_adjacent != 0, legacy);
}

template <bool HAS_NAN, bool LEAF_OUT, class Src>
static void launch_tiled(const PredictArgs& a, const Src& src, const PredictPlan& plan, cudaStream_t s) {
  static bool attr = false;
  if (!attr) { CUDA_OK(cudaFuncSetAttribute(predict_tiled_kernel<HAS_NAN, LEAF_OUT, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPredictSmem)); attr = true; }
  for (const PredictChunk& ch : plan.chunks) {
    const int rows = ch.rows, threads = ch.threads;
    const int64_t tiles = (a.n + rows - 1) / rows;
    const int grid = (int)std::min<int64_t>(tiles, engine_num_sms() * (threads == 1024 ? 1 : 2048 / threads));
    predict_tiled_kernel<HAS_NAN, LEAF_OUT, Src><<<grid, threads, ch.smem, s>>>(a, src, ch.tree_lo, ch.tree_hi, plan.pitch, rows, tiles);
    ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  }
}

// executes plan_for(a): one tiled launch per tree chunk, or the thread-per-row kernel
void launch_predict(const PredictArgs& a, cudaStream_t s) {
  if (a.n == 0 || a.tree_end <= a.tree_begin) return;
  const PredictPlan plan = plan_for(a);
  const RowsF32 src{a.X, a.F};
  if (plan.kernel == PredictKernel::kTiled) {
    if (a.leaf) { if (a.has_nan) launch_tiled<true, true>(a, src, plan, s); else launch_tiled<false, true>(a, src, plan, s); }
    else { if (a.has_nan) launch_tiled<true, false>(a, src, plan, s); else launch_tiled<false, false>(a, src, plan, s); }
    return;
  }
  predict_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, s>>>(a, src); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// plan_for(a) on the in-place input d (a.X unused, a.F == d.F): the NaN-aware tiled kernel, or thread-per-row, reading d
template <class Src>
static void launch_predict_src(const PredictArgs& a, const Src& src, cudaStream_t s) {
  const PredictPlan plan = plan_for(a);
  if (plan.kernel == PredictKernel::kTiled) { launch_tiled<true, false>(a, src, plan, s); return; }
  predict_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, s>>>(a, src); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_predict_inplace(const PredictArgs& a, const InputDesc& d, cudaStream_t s) {
  B200_CHECK(a.leaf == nullptr && a.F == d.F && a.n == d.n, "launch_predict_inplace: margins of the input's rows only");
  if (a.n == 0 || a.tree_end <= a.tree_begin) return;
  if (d.indptr) { launch_predict_src(a, CsrSrc{d}, s); return; }
  switch (d.type) {
    case kInF32: launch_predict_src(a, StridedSrc<kInF32>{d}, s); return;
    case kInF64: launch_predict_src(a, StridedSrc<kInF64>{d}, s); return;
    case kInF16: launch_predict_src(a, StridedSrc<kInF16>{d}, s); return;
    default: throw Error("launch_predict_inplace: element type " + std::to_string(d.type) + " is converted to float32 first (launch_convert_rows)");
  }
}

// rows [r0, r0 + rows) of d as float32 into out (row-major, rows x d.F, NaN = missing)
__global__ void __launch_bounds__(256) convert_rows_kernel(InputDesc d, int64_t r0, int64_t rows, float* out) {
  const int F = d.F;
  const int64_t total = rows * F;
  const bool rows_fast = (d.s0 < 0 ? -d.s0 : d.s0) < (d.s1 < 0 ? -d.s1 : d.s1);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r; int f;
    if (rows_fast) { f = (int)(i / rows); r = i - (int64_t)f * rows; } else { r = i / F; f = (int)(i - r * F); }
    out[r * F + f] = load_x(d, r0 + r, f);
  }
}
void launch_convert_rows(const InputDesc& d, int64_t r0, int64_t rows, float* out, cudaStream_t s) {
  if (rows * d.F <= 0) return;
  convert_rows_kernel<<<grid_for(rows * d.F, 256, engine_num_sms() * 16), 256, 0, s>>>(d, r0, rows, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_transform(float* m, int64_t n, int K, int objective, float* out_class, cudaStream_t s) {
  if (n == 0) return;
  transform_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(m, n, K, objective, out_class); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_curve_scores(const float* margin, int64_t n, int K, int c, int logistic, float* key, int* iota, cudaStream_t s) {
  if (n == 0) return;
  curve_scores_kernel<<<grid_for(n), 256, 0, s>>>(margin, n, K, c, logistic, key, iota); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_fill(float* p, int64_t n, float v, cudaStream_t s) {
  if (n == 0) return;
  fill_kernel<<<grid_for(n), 256, 0, s>>>(p, n, v); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_metric(const MetricArgs& a, cudaStream_t s) {
  if (a.n == 0) return;
  metric_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
