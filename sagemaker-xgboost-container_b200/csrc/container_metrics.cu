// container_metrics.cu -- the container's own metrics from the prediction cache (DESIGN.md "Container metrics").
//
// One pass over the rows reads each row's margins and label once and applies predict()'s transform (transform.h).  The
// classification metrics get an exact integer confusion matrix of (label, predicted class): block-private shared-memory
// counts, flushed with integer atomics.  The regression metrics get float32 elementwise terms, summed in numpy's pairwise
// order (PairwisePlan): the blocks of at most 128 terms in parallel, then the joins level by level (wide levels one
// launch each, the narrow top levels in one CTA).  No
// floating-point atomics anywhere, so every result is the same from run to run and equals numpy's float32 sum bit for bit.
//
// Built with the default flags like misc.cu, so the transform's expf rounds like predict()'s; the metric arithmetic uses
// __fmul_rn / __fadd_rn, which are never fused, so it rounds like numpy's.
#include <algorithm>
#include <climits>
#include "container_metrics.h"
#include "transform.h"          // with misc.cu's flags (build.py): the transform rounds like predict()'s

namespace b200 {

namespace {

constexpr int kLeafMax = 128;             // numpy's PW_BLOCKSIZE
constexpr int kRowThreads = 256, kCombineThreads = 1024;

int grid_for(int64_t n, int cap) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + kRowThreads - 1) / kRowThreads, cap)); }

// the value predict() returns for a row (one output per row)
__device__ __forceinline__ float row_value(const float* m, int K, int objective, int output_margin) {
  if (output_margin) return m[0];
  if (objective == kSoftmax) return (float)softmax_class(m, K);
  if (objective == kSoftprob) { float wmax; const float wsum = softmax_sum(m, K, &wmax); return expf(m[0] - wmax) / wsum; }
  return transform_one(m[0], objective);
}

// cols == 1: pred class = value > 0 (the container's margin_to_class_label on 1-D predictions); cols > 1: np.argmax over the
// row's predict() values, the first largest and a NaN first of all.  Regression terms (y - p)^2 and |y - p| for cols == 1.
// out[0] |= 1: a label the confusion matrix cannot hold; |= 2: a non-finite label, prediction or squared error.
__global__ void __launch_bounds__(kRowThreads) container_rows_kernel(ContainerArgs a, int cols, int P, float* terms, long long* out) {
  extern __shared__ unsigned cnt[];
  const int ncnt = a.want_class ? kContainerLabels * P : 0;
  for (int i = threadIdx.x; i < ncnt; i += blockDim.x) cnt[i] = 0;
  __syncthreads();
  unsigned bad = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float y = a.label[r];
    const float* m = a.margin + r * a.K;
    float v = 0.0f; int pc = 0;
    if (cols == 1) {
      v = row_value(m, a.K, a.objective, a.output_margin);
      pc = v > 0.0f ? 1 : 0;
    } else if (a.want_class) {
      const bool prob = !a.output_margin && a.objective == kSoftprob;
      float wmax = 0.0f, wsum = 1.0f;
      if (prob) wsum = softmax_sum(m, a.K, &wmax);
      float best = 0.0f;
      for (int k = 0; k < cols; ++k) {
        const float x = prob ? expf(m[k] - wmax) / wsum : m[k];
        if (isnan(x)) { pc = k; break; }
        if (k == 0 || x > best) { best = x; pc = k; }
      }
    }
    if (a.want_class) {
      if (y >= 0.0f && y < (float)kContainerLabels && y == floorf(y)) atomicAdd(&cnt[(int)y * P + pc], 1u);
      else bad |= 1u;
    }
    if (a.want_reg) {
      const float d = y - v, sq = __fmul_rn(d, d);
      terms[r] = sq; terms[a.n + r] = fabsf(d);
      if (!isfinite(y) || !isfinite(v) || !isfinite(sq)) bad |= 2u;
    }
  }
  bad = __reduce_or_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0 && bad) atomicOr((unsigned long long*)out, (unsigned long long)bad);
  __syncthreads();
  for (int i = threadIdx.x; i < ncnt; i += blockDim.x)
    if (cnt[i]) atomicAdd((unsigned long long*)out + kContainerOutHead + i, (unsigned long long)cnt[i]);
}

// (y - mean)^2 with mean = float32(double(sum y) / n), as numpy's float32 mean divides
__global__ void __launch_bounds__(kRowThreads) deviation_terms_kernel(const float* y, int64_t n, const float* sum_y, float* out) {
  const float mean = (float)((double)*sum_y / (double)n);
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const float d = y[r] - mean;
    out[r] = __fmul_rn(d, d);
  }
}

// one block of numpy's pairwise_sum per thread and term array
__global__ void __launch_bounds__(kRowThreads) pairwise_leaf_kernel(const float* terms, int64_t tstride, int nterms, const int2* leaf, int leaves,
                                                                    float* vals, int64_t vstride) {
  const int64_t total = (int64_t)leaves * nterms;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / leaves), l = (int)(i % leaves);
    const int2 b = leaf[l];
    const float* x = terms + t * tstride + b.x;
    float res;
    if (b.y < 8) {
      res = 0.0f;
      for (int j = 0; j < b.y; ++j) res = __fadd_rn(res, x[j]);
    } else {
      float r[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) r[k] = x[k];
      int j = 8;
      for (; j < b.y - b.y % 8; j += 8) {
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] = __fadd_rn(r[k], x[j + k]);
      }
      res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
      for (; j < b.y; ++j) res = __fadd_rn(res, x[j]);
    }
    vals[t * vstride + l] = res;
  }
}

// the joins of levels [h0, h1) of the recursion, lowest first, from op `begin` on; a level only reads nodes of lower levels, so
// one level may run on any grid, several levels only on one CTA (a __syncthreads between levels)
__global__ void __launch_bounds__(kCombineThreads) pairwise_combine_kernel(float* vals, int64_t vstride, int nterms, int leaves, const int2* ops,
                                                                           const int* level_end, int h0, int h1, int begin) {
  for (int h = h0; h < h1; ++h) {
    const int end = level_end[h];
    for (int j = begin + blockIdx.x * blockDim.x + threadIdx.x; j < end; j += gridDim.x * blockDim.x) {
      const int2 o = ops[j];
      for (int t = 0; t < nterms; ++t) { float* v = vals + t * vstride; v[leaves + j] = __fadd_rn(v[o.x], v[o.y]); }
    }
    begin = end;
    __syncthreads();
  }
}

// node id and height of the subtree over terms [start, start + m)
struct BuildNode { int l, r, h; };
int plan_node(int64_t start, int64_t m, std::vector<int2>* leaves, std::vector<BuildNode>* inner, int* height) {
  if (m <= kLeafMax) { leaves->push_back(make_int2((int)start, (int)m)); *height = 0; return (int)leaves->size() - 1; }
  int64_t n2 = m / 2; n2 -= n2 % 8;
  int hl, hr;
  const int l = plan_node(start, n2, leaves, inner, &hl), r = plan_node(start + n2, m - n2, leaves, inner, &hr);
  inner->push_back({l, r, std::max(hl, hr) + 1});
  *height = std::max(hl, hr) + 1;
  return -(int)inner->size();            // inner node k is -(k + 1) until the ids are final
}

// sums the terms [t][0, n) of nterms arrays in numpy's order; sums of array t end at vals[t * vstride + plan.nodes() - 1]
void pairwise_sums(const float* terms, int64_t tstride, int nterms, const PairwisePlan& plan, float* vals, int64_t vstride, cudaStream_t s) {
  const int64_t leaf_threads = (int64_t)plan.leaves * nterms;
  pairwise_leaf_kernel<<<grid_for(leaf_threads, engine_num_sms() * 8), kRowThreads, 0, s>>>(terms, tstride, nterms, plan.d_leaf.p, plan.leaves, vals, vstride);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  // the wide lower levels one launch each over the whole GPU, the narrow top levels together on one CTA
  const int levels = (int)plan.level_end.size();
  int h = 0, begin = 0;
  for (; h < levels && plan.level_end[h] - begin > 4 * kCombineThreads; begin = plan.level_end[h++]) {
    const int grid = (int)std::min<int64_t>((plan.level_end[h] - begin + kCombineThreads - 1) / kCombineThreads, engine_num_sms() * 2);
    pairwise_combine_kernel<<<grid, kCombineThreads, 0, s>>>(vals, vstride, nterms, plan.leaves, plan.d_ops.p, plan.d_level_end.p, h, h + 1, begin);
    ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  }
  if (h == levels) return;
  pairwise_combine_kernel<<<1, kCombineThreads, 0, s>>>(vals, vstride, nterms, plan.leaves, plan.d_ops.p, plan.d_level_end.p, h, levels, begin);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace

void PairwisePlan::build(int64_t count, cudaStream_t s) {
  if (n == count) return;
  B200_CHECK(count > 0 && count <= INT_MAX, "pairwise plan: row count out of range");
  std::vector<int2> leaf; std::vector<BuildNode> inner; int h;
  const int root = plan_node(0, count, &leaf, &inner, &h);
  (void)root;
  leaves = (int)leaf.size();
  // order the inner nodes by height (stable), then give node leaves + j to the j-th of them
  std::vector<int> order(inner.size());
  for (size_t k = 0; k < order.size(); ++k) order[k] = (int)k;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return inner[a].h < inner[b].h; });
  std::vector<int> final_id(inner.size());
  for (size_t j = 0; j < order.size(); ++j) final_id[order[j]] = leaves + (int)j;
  auto id = [&](int v) { return v >= 0 ? v : final_id[-v - 1]; };
  std::vector<int2> ops(inner.size());
  level_end.clear();
  for (size_t j = 0; j < order.size(); ++j) {
    const BuildNode& b = inner[order[j]];
    ops[j] = make_int2(id(b.l), id(b.r));
    if ((int)level_end.size() < b.h) level_end.resize(b.h, (int)j);
    level_end[b.h - 1] = (int)j + 1;
  }
  d_leaf.alloc(leaf.size()); d_ops.alloc(std::max<size_t>(ops.size(), 1)); d_level_end.alloc(std::max<size_t>(level_end.size(), 1));
  CUDA_OK(cudaMemcpyAsync(d_leaf.p, leaf.data(), sizeof(int2) * leaf.size(), cudaMemcpyHostToDevice, s));
  if (!ops.empty()) CUDA_OK(cudaMemcpyAsync(d_ops.p, ops.data(), sizeof(int2) * ops.size(), cudaMemcpyHostToDevice, s));
  if (!level_end.empty()) CUDA_OK(cudaMemcpyAsync(d_level_end.p, level_end.data(), sizeof(int) * level_end.size(), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaStreamSynchronize(s));      // the host vectors go out of scope
  n = count;
}

void ContainerScratch::ensure(int64_t term_count, int64_t val_count) {
  terms.ensure((size_t)term_count); vals.ensure((size_t)val_count); out.ensure(kContainerOutLen);
}

void container_metrics_device(const ContainerArgs& a, ContainerSums* dm_sums, ContainerScratch* sc, cudaStream_t s) {
  const int cols = (!a.output_margin && a.objective == kSoftmax) ? 1 : a.K;
  const int P = cols == 1 ? 2 : cols;
  const bool reg = a.want_reg != 0;
  PairwisePlan& plan = dm_sums->plan;
  if (reg) plan.build(a.n, s);
  // n-sized term arrays only for what is asked: (y - p)^2 and |y - p|, and r2's (y - mean)^2 while its label sums are built
  const bool label_pass = a.want_r2 && !dm_sums->labels_valid;
  sc->ensure(reg ? a.n * (label_pass ? 3 : 2) : 0, reg ? (int64_t)plan.nodes() * 2 : 0);
  CUDA_OK(cudaMemsetAsync(sc->out.p, 0, sizeof(long long) * (kContainerOutHead + (size_t)kContainerLabels * P), s));
  const int64_t vstride = reg ? plan.nodes() : 0;
  const int root = reg ? plan.nodes() - 1 : 0;
  if (label_pass) {
    // labels only: sum y, then sum (y - mean)^2, kept on the matrix until its labels change
    dm_sums->label_sums.ensure(2);
    pairwise_sums(a.label, 0, 1, plan, sc->vals.p, vstride, s);
    CUDA_OK(cudaMemcpyAsync(dm_sums->label_sums.p, sc->vals.p + root, sizeof(float), cudaMemcpyDeviceToDevice, s));
    float* dev = sc->terms.p + 2 * a.n;
    deviation_terms_kernel<<<grid_for(a.n, engine_num_sms() * 8), kRowThreads, 0, s>>>(a.label, a.n, dm_sums->label_sums.p, dev);
    ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    pairwise_sums(dev, 0, 1, plan, sc->vals.p, vstride, s);
    CUDA_OK(cudaMemcpyAsync(dm_sums->label_sums.p + 1, sc->vals.p + root, sizeof(float), cudaMemcpyDeviceToDevice, s));
    dm_sums->labels_valid = true;
  }
  const size_t smem = a.want_class ? sizeof(unsigned) * kContainerLabels * P : 0;
  container_rows_kernel<<<grid_for(a.n, engine_num_sms() * 8), kRowThreads, smem, s>>>(a, cols, P, sc->terms.p, sc->out.p);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  if (reg) {
    pairwise_sums(sc->terms.p, a.n, 2, plan, sc->vals.p, vstride, s);
    // float bits into the low half of out[4], out[5] (little-endian); the high halves stay zero
    CUDA_OK(cudaMemcpyAsync(sc->out.p + 4, sc->vals.p + root, sizeof(float), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(sc->out.p + 5, sc->vals.p + vstride + root, sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  if (a.want_r2) {
    CUDA_OK(cudaMemcpyAsync(sc->out.p + 6, dm_sums->label_sums.p, sizeof(float), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(sc->out.p + 7, dm_sums->label_sums.p + 1, sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
}

}  // namespace b200
