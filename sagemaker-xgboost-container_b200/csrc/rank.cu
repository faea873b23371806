// rank.cu -- rank:pairwise, rank:ndcg and rank:map: LambdaRank gradient pairs over the topk pairs of each query group, and the
// ndcg / map metrics.  Restates upstream xgboost src/objective/lambdarank_obj.{cc,cu} and src/metric/rank_metric.cc
// [UPSTREAM-RECALL]; DESIGN.md "Learning to rank" gives the formulas and which details rest on recall.
//
// Determinism: no floating-point atomics.  Every document gathers its own pairs (one warp per document, lane l takes the partners
// l, l + 32, ...), sums them in double and reduces the lanes with a fixed butterfly; every per-group sum is one warp per group
// in the same way.  The float gradients therefore depend only on the inputs, not on the launch configuration or group order.
// Compiled with --fmad=false (build.py) so the double arithmetic rounds like a host restatement of the same expressions.
#include <cub/cub.cuh>
#include "rank.h"
#include "rng.h"

namespace b200 {

constexpr int kThreads = 256, kWarps = kThreads / 32;

static int blocks_for(int64_t items, int per_block) {
  int64_t g = (items + per_block - 1) / per_block;
  const int64_t cap = (int64_t)engine_num_sms() * 16;
  return (int)std::max<int64_t>(1, std::min(g, cap));
}

__device__ __forceinline__ double gain(float y, int exp_gain) { return exp_gain ? exp2((double)y) - 1.0 : (double)y; }
__device__ __forceinline__ double discount(int r) { return 1.0 / log2((double)r + 2.0); }
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// group layout
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) row_group_kernel(const int* ptr, int64_t G, int64_t n, int* row_group) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = G;                  // the last group g with ptr[g] <= r (empty groups are skipped)
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (ptr[mid] <= r) lo = mid; else hi = mid; }
    row_group[r] = (int)lo;
  }
}

template <class T>
static void segmented_sort_desc(const float* key_in, float* key_out, const T* val_in, T* val_out, int64_t n, const RankGroups& rg,
                                RankScratch* sc, cudaStream_t s) {
  size_t bytes = 0;
  if (rg.G == 1) {           // one group (a matrix without groups): a device-wide stable radix sort, not one CTA on the whole segment
    if (val_in) {
      CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(nullptr, bytes, key_in, key_out, val_in, val_out, (int)n, 0, 32, s));
      sc->tmp.ensure(std::max<size_t>(bytes, 1));
      CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(sc->tmp.p, bytes, key_in, key_out, val_in, val_out, (int)n, 0, 32, s));
    } else {
      CUDA_OK(cub::DeviceRadixSort::SortKeysDescending(nullptr, bytes, key_in, key_out, (int)n, 0, 32, s));
      sc->tmp.ensure(std::max<size_t>(bytes, 1));
      CUDA_OK(cub::DeviceRadixSort::SortKeysDescending(sc->tmp.p, bytes, key_in, key_out, (int)n, 0, 32, s));
    }
  } else if (val_in) {
    CUDA_OK(cub::DeviceSegmentedSort::StableSortPairsDescending(nullptr, bytes, key_in, key_out, val_in, val_out, (int)n, (int)rg.G, rg.ptr.p, rg.ptr.p + 1, s));
    sc->tmp.ensure(std::max<size_t>(bytes, 1));
    CUDA_OK(cub::DeviceSegmentedSort::StableSortPairsDescending(sc->tmp.p, bytes, key_in, key_out, val_in, val_out, (int)n, (int)rg.G, rg.ptr.p, rg.ptr.p + 1, s));
  } else {
    CUDA_OK(cub::DeviceSegmentedSort::StableSortKeysDescending(nullptr, bytes, key_in, key_out, (int)n, (int)rg.G, rg.ptr.p, rg.ptr.p + 1, s));
    sc->tmp.ensure(std::max<size_t>(bytes, 1));
    CUDA_OK(cub::DeviceSegmentedSort::StableSortKeysDescending(sc->tmp.p, bytes, key_in, key_out, (int)n, (int)rg.G, rg.ptr.p, rg.ptr.p + 1, s));
  }
  ++g_kernel_launches;
}

__global__ void __launch_bounds__(kThreads) iota_kernel(int64_t n, int* iota) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) iota[i] = (int)i;
}

void rank_groups_build(const std::vector<unsigned>& group_ptr, const float* label, int64_t n, RankGroups* rg, RankScratch* sc, cudaStream_t s) {
  B200_CHECK(n < (int64_t)0x7fffffff, "ranking: more than 2^31-1 rows");
  std::vector<int> ptr;
  if (group_ptr.empty()) ptr = {0, (int)n};
  else ptr.assign(group_ptr.begin(), group_ptr.end());
  B200_CHECK(ptr.back() == n, "ranking: the query groups do not cover the rows");
  rg->G = (int64_t)ptr.size() - 1; rg->n = n;
  rg->ptr.alloc(ptr.size()); rg->row_group.alloc(std::max<int64_t>(n, 1)); rg->ideal.alloc(std::max<int64_t>(n, 1)); rg->ideal_order.alloc(std::max<int64_t>(n, 1));
  CUDA_OK(cudaMemcpyAsync(rg->ptr.p, ptr.data(), sizeof(int) * ptr.size(), cudaMemcpyHostToDevice, s));
  if (n) {
    row_group_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(rg->ptr.p, rg->G, n, rg->row_group.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    sc->iota.ensure(n);
    iota_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(n, sc->iota.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    segmented_sort_desc<int>(label, rg->ideal.p, sc->iota.p, rg->ideal_order.p, n, *rg, sc, s);
  }
  CUDA_OK(cudaStreamSynchronize(s));      // the host pointer array is released on return
  rg->valid = true;
}

// ---------------------------------------------------------------------------------------------
// the margins in sorted order: stable, descending, -0.0 read as +0.0, ties in row order
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) key_kernel(const float* m, int64_t n, float* key, int* iota) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = m[i];
    key[i] = v == 0.0f ? 0.0f : v; iota[i] = (int)i;
  }
}
__global__ void __launch_bounds__(kThreads) gather_labels_kernel(const float* y, const int* order, int64_t n, float* ys) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) ys[p] = y[order[p]];
}

static void rank_sort(const float* margin, const float* label, const RankGroups& rg, RankScratch* sc, cudaStream_t s) {
  const int64_t n = rg.n;
  sc->key.ensure(n); sc->key_sorted.ensure(n); sc->y_sorted.ensure(n); sc->iota.ensure(n); sc->order.ensure(n);
  key_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(margin, n, sc->key.p, sc->iota.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  segmented_sort_desc<int>(sc->key.p, sc->key_sorted.p, sc->iota.p, sc->order.p, n, rg, sc, s);
  gather_labels_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(label, sc->order.p, n, sc->y_sorted.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// per-group passes: one warp per group
// ---------------------------------------------------------------------------------------------
#define FOR_EACH_GROUP_WARP(G) \
  const int lane = threadIdx.x & 31; \
  for (int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < (G); g += ((int64_t)gridDim.x * blockDim.x) >> 5)

// MAP: inclusive (hits, sum of 1 / (r + 1) over the hits) at every position r of the group, in the current order
__global__ void __launch_bounds__(kThreads) map_prefix_kernel(const float* ys, const int* ptr, int64_t G, double2* hq) {
  FOR_EACH_GROUP_WARP(G) {
    const int b = ptr[g], e = ptr[g + 1];
    double ch = 0.0, cq = 0.0;
    for (int base = b; base < e; base += 32) {
      const int p = base + lane;
      const bool rel = p < e && ys[p] > 0.0f;
      double h = rel ? 1.0 : 0.0, q = rel ? 1.0 / (double)(p - b + 1) : 0.0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double th = __shfl_up_sync(0xffffffffu, h, o), tq = __shfl_up_sync(0xffffffffu, q, o);
        if (lane >= o) { h += th; q += tq; }
      }
      if (p < e) hq[p] = make_double2(ch + h, cq + q);
      ch += __shfl_sync(0xffffffffu, h, 31); cq += __shfl_sync(0xffffffffu, q, 31);
    }
  }
}

// 1 / IDCG over the first min(k, n) label-sorted positions (0 when IDCG = 0)
__global__ void __launch_bounds__(kThreads) inv_idcg_kernel(const float* ideal, const int* ptr, int64_t G, int k, int exp_gain, double* out) {
  FOR_EACH_GROUP_WARP(G) {
    const int b = ptr[g], n = ptr[g + 1] - b, kk = min(k, n);
    double v = 0.0;
    for (int j = lane; j < kk; j += 32) v += gain(ideal[b + j], exp_gain) * discount(j);
    v = warp_sum(v);
    if (lane == 0) out[g] = v == 0.0 ? 0.0 : 1.0 / v;
  }
}

// each group's factor: log2(1 + S) / S with S the sum of |lambda| over its documents (lambdarank_normalization), times w_g * wscale
__global__ void __launch_bounds__(kThreads) group_scale_kernel(const double* lam, const int* ptr, int64_t G, int normalization, const float* w,
                                                               double wscale, double* out) {
  FOR_EACH_GROUP_WARP(G) {
    const int b = ptr[g], e = ptr[g + 1];
    double S = 0.0;
    for (int p = b + lane; p < e; p += 32) S += lam[p];
    S = warp_sum(S);
    const double norm = normalization && S > 0.0 ? log2(1.0 + S) / S : 1.0;
    if (lane == 0) out[g] = norm * (w ? (double)w[g] * wscale : 1.0);
  }
}

// ---------------------------------------------------------------------------------------------
// the pairs of one document, one warp per document (position p of the sorted order)
// ---------------------------------------------------------------------------------------------
struct PairArgs {
  const float* ks; const float* ys; const double2* hq; const int* ptr; const int* row_group; const double* inv_idcg;
  double* acc;                          // [3][n]: sum of g, of h, of |lambda| per position
  int64_t n; int objective, k, exp_gain, score_normalization;
};

// |delta AP| * R when the documents at positions a < b (one relevant, one not) swap; hq holds the group's inclusive prefixes
__device__ __forceinline__ double map_delta(int a, int b, bool rel_a, const double2* hq_group) {
  const double2 A = hq_group[a], B = hq_group[b];
  const double ia = 1.0 / (double)(a + 1), ib = 1.0 / (double)(b + 1);
  if (rel_a) return fabs(B.x * ib - A.x * ia - (B.y - A.y));            // the relevant document moves down from a to b
  return fabs((A.x + 1.0) * ia - B.x * ib + (B.y - ib - A.y));          // it moves up from b to a
}

// (lambda, h) of one pair with labels y_high > y_low at positions r_high, r_low of the group's margin order, gains and discounts
// given; the group's constants in d
struct PairTerms { double lam, h; };
__device__ __forceinline__ PairTerms pair_terms(const PairArgs& d, int b, double inv, double R, bool snorm, double g_high, double g_low,
                                                int r_high, int r_low, bool rel_first, double s_high, double s_low) {
  double delta = 1.0;
  if (d.objective == kRankNdcg) delta = fabs((g_high - g_low) * (discount(r_high) - discount(r_low))) * inv;
  else if (d.objective == kRankMap) delta = map_delta(min(r_high, r_low), max(r_high, r_low), rel_first, d.hq + b) / R;
  if (snorm) delta /= fabs(s_high - s_low) + 0.01;
  const double sigma = 1.0 / (1.0 + exp(-(s_high - s_low)));
  PairTerms t;
  t.lam = (sigma - 1.0) * delta;
  t.h = fmax(sigma * (1.0 - sigma), 1e-16) * delta * 2.0;
  return t;
}

__global__ void __launch_bounds__(kThreads) rank_pairs_kernel(PairArgs d) {
  const int lane = threadIdx.x & 31;
  for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < d.n; p += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int g = d.row_group[p], b = d.ptr[g], e = d.ptr[g + 1], n = e - b, lp = (int)(p - b);
    const int kk = min(d.k, n);
    const int m = lp < kk ? n : kk;      // position p < K pairs with every other position, p >= K with the positions < K
    const float yp = d.ys[p];
    const double sp = (double)d.ks[p];
    const bool snorm = d.score_normalization && d.ks[b] != d.ks[e - 1];
    const double inv = d.objective == kRankNdcg ? d.inv_idcg[g] : 0.0;
    const double R = d.objective == kRankMap ? d.hq[e - 1].x : 1.0;
    const double gp = d.objective == kRankNdcg ? gain(yp, d.exp_gain) : 0.0;
    double sg = 0.0, sh = 0.0, sl = 0.0;
    for (int q = lane; q < m; q += 32) {
      if (q == lp) continue;
      const float yq = d.ys[b + q];
      if (yq == yp) continue;
      const bool high = yp > yq;
      const double gq = d.objective == kRankNdcg ? gain(yq, d.exp_gain) : 0.0;
      const double sq = (double)d.ks[b + q];
      const bool rel_first = ((lp < q) ? yp : yq) > 0.0f;
      const PairTerms t = high ? pair_terms(d, b, inv, R, snorm, gp, gq, lp, q, rel_first, sp, sq)
                               : pair_terms(d, b, inv, R, snorm, gq, gp, q, lp, rel_first, sq, sp);
      sg += high ? t.lam : -t.lam; sh += t.h; sl -= t.lam;
    }
    sg = warp_sum(sg); sh = warp_sum(sh); sl = warp_sum(sl);
    if (lane == 0) { d.acc[p] = sg; d.acc[d.n + p] = sh; d.acc[2 * d.n + p] = sl; }
  }
}

// ---------------------------------------------------------------------------------------------
// lambdarank_pair_method=mean: each document, taken in the label order of its group, draws k partners uniformly from the documents
// outside its label bucket.  A pair adds to both documents, so the sums are int64 fixed point (2^-32) with integer atomics:
// integer addition is associative, so the sums do not depend on the order the pairs arrive in.
// ---------------------------------------------------------------------------------------------
constexpr double kFixScale = 4294967296.0;
__device__ __forceinline__ void fix_add(unsigned long long* a, double v) { atomicAdd(a, (unsigned long long)llrint(v * kFixScale)); }

__global__ void __launch_bounds__(kThreads) position_kernel(const int* order, int64_t n, int* pos) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) pos[order[p]] = (int)p;
}

struct MeanArgs {
  PairArgs d; const float* ideal; const int* ideal_order; const int* pos; unsigned long long* fix;
  int64_t row_offset; unsigned seed; unsigned long long stream;
};

__global__ void __launch_bounds__(kThreads) rank_mean_kernel(MeanArgs a) {
  const PairArgs& d = a.d;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < d.n; q += (int64_t)gridDim.x * blockDim.x) {
    const int g = d.row_group[q], b = d.ptr[g], e = d.ptr[g + 1];
    const float yi = a.ideal[q];
    int lo = b, hi = e;                  // the bucket [bl, bh) of yi in the descending labels of the group
    { int l = b, r = e; while (l < r) { const int m = (l + r) >> 1; if (a.ideal[m] > yi) l = m + 1; else r = m; } lo = l; }
    { int l = lo, r = e; while (l < r) { const int m = (l + r) >> 1; if (a.ideal[m] >= yi) l = m + 1; else r = m; } hi = l; }
    const int c = (e - b) - (hi - lo);
    if (c == 0) continue;
    const int row_i = a.ideal_order[q], pi = a.pos[row_i];
    const bool snorm = d.score_normalization && d.ks[b] != d.ks[e - 1];
    const double inv = d.objective == kRankNdcg ? d.inv_idcg[g] : 0.0;
    const double R = d.objective == kRankMap ? d.hq[e - 1].x : 1.0;
    const double gi = d.objective == kRankNdcg ? gain(yi, d.exp_gain) : 0.0, si = (double)d.ks[pi];
    for (int j = 0; j < d.k; ++j) {
      const float u = rng_uniform(a.seed, a.stream + (unsigned long long)j, (unsigned long long)(row_i + a.row_offset));
      const int t = min(c - 1, (int)((double)u * (double)c));
      const int jq = b + (t < lo - b ? t : t + (hi - lo));
      const int pj = a.pos[a.ideal_order[jq]];
      const float yj = a.ideal[jq];
      const bool high = yi > yj;
      const double gj = d.objective == kRankNdcg ? gain(yj, d.exp_gain) : 0.0, sj = (double)d.ks[pj];
      const int ri = pi - b, rj = pj - b;
      const bool rel_first = ((ri < rj) ? yi : yj) > 0.0f;
      const PairTerms pt = high ? pair_terms(d, b, inv, R, snorm, gi, gj, ri, rj, rel_first, si, sj)
                                : pair_terms(d, b, inv, R, snorm, gj, gi, rj, ri, rel_first, sj, si);
      const int ph = high ? pi : pj, pl = high ? pj : pi;
      fix_add(a.fix + ph, pt.lam); fix_add(a.fix + pl, -pt.lam);
      fix_add(a.fix + d.n + pi, pt.h); fix_add(a.fix + d.n + pj, pt.h);
      fix_add(a.fix + 2 * d.n + pi, -pt.lam); fix_add(a.fix + 2 * d.n + pj, -pt.lam);
    }
  }
}

__global__ void __launch_bounds__(kThreads) unfix_kernel(const unsigned long long* fix, int64_t n, double* acc) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) acc[i] = (double)(long long)fix[i] / kFixScale;
}

__device__ __forceinline__ void fold_absmax(float mg, float mh, unsigned* absmax) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  __shared__ float sg[kWarps], sh[kWarps];
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kWarps; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
    if (absmax) { atomicMax(absmax, __float_as_uint(mg)); atomicMax(absmax + 1, __float_as_uint(mh)); }
  }
}

// (g, h) of each document: its pair sums times its group's factor, rounded to float once, written to its row
__global__ void __launch_bounds__(kThreads) rank_write_kernel(RankGradArgs a, const int* order, const int* row_group, const double* acc, const double* scale) {
  float mg = 0.f, mh = 0.f;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = order[p];
    const double f = scale[row_group[p]];
    float gf = (float)(acc[p] * f), hf = (float)(acc[a.n + p] * f);
    if (a.subsample < 1.0f && !(rng_uniform(a.seed, 0x2000ull + a.iter, (unsigned long long)(r + a.row_offset)) < a.subsample)) { gf = 0.f; hf = 0.f; }
    a.gpair[r] = make_float2(gf, hf);
    mg = fmaxf(mg, fabsf(gf)); mh = fmaxf(mh, hf);
  }
  fold_absmax(mg, mh, a.absmax);
}

void launch_rank_gradient(const RankGradArgs& a, const RankGroups& rg, RankScratch* sc, cudaStream_t s) {
  if (a.n == 0) return;
  B200_CHECK(rg.valid && rg.n == a.n, "ranking: the query groups do not match the matrix");
  const int64_t n = a.n, G = rg.G;
  rank_sort(a.margin, a.label, rg, sc, s);
  sc->acc.ensure(3 * (size_t)n); sc->group.ensure((size_t)G);
  PairArgs d{}; d.ks = sc->key_sorted.p; d.ys = sc->y_sorted.p; d.ptr = rg.ptr.p; d.row_group = rg.row_group.p; d.acc = sc->acc.p;
  d.n = n; d.objective = a.objective; d.k = a.k; d.exp_gain = a.exp_gain; d.score_normalization = a.score_normalization;
  if (a.objective == kRankMap) {
    sc->hq.ensure(n);
    map_prefix_kernel<<<blocks_for(G * 32, kThreads), kThreads, 0, s>>>(sc->y_sorted.p, rg.ptr.p, G, sc->hq.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    d.hq = sc->hq.p;
  }
  if (a.objective == kRankNdcg) {
    const int idcg_k = a.mean ? 0x7fffffff : a.k;          // IDCG over the whole group under mean, over the top K under topk
    inv_idcg_kernel<<<blocks_for(G * 32, kThreads), kThreads, 0, s>>>(rg.ideal.p, rg.ptr.p, G, idcg_k, a.exp_gain, sc->group.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    d.inv_idcg = sc->group.p;
  }
  if (!a.mean) {
    rank_pairs_kernel<<<blocks_for(n * 32, kThreads), kThreads, 0, s>>>(d); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  } else {
    sc->pos.ensure(n); sc->fix.ensure(3 * (size_t)n);
    CUDA_OK(cudaMemsetAsync(sc->fix.p, 0, sizeof(unsigned long long) * 3 * n, s));
    position_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(sc->order.p, n, sc->pos.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    MeanArgs ma{}; ma.d = d; ma.ideal = rg.ideal.p; ma.ideal_order = rg.ideal_order.p; ma.pos = sc->pos.p; ma.fix = sc->fix.p;
    ma.row_offset = a.row_offset; ma.seed = a.seed; ma.stream = a.pair_stream;
    rank_mean_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(ma); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    unfix_kernel<<<blocks_for(3 * n, kThreads), kThreads, 0, s>>>(sc->fix.p, 3 * n, sc->acc.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  }
  group_scale_kernel<<<blocks_for(G * 32, kThreads), kThreads, 0, s>>>(sc->acc.p + 2 * n, rg.ptr.p, G, a.normalization, a.weight, a.wscale, sc->group.p);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  rank_write_kernel<<<blocks_for(n, kThreads), kThreads, 0, s>>>(a, sc->order.p, rg.row_group.p, sc->acc.p, sc->group.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// metrics
// ---------------------------------------------------------------------------------------------
// v_g and w_g of every group into out[g] and out[G + g]
__global__ void __launch_bounds__(kThreads) rank_metric_kernel(const float* ys, const float* ideal, const int* ptr, int64_t G, int map, int k,
                                                               int exp_gain, int minus, const float* w, double* out) {
  FOR_EACH_GROUP_WARP(G) {
    const int b = ptr[g], n = ptr[g + 1] - b, kk = k > 0 ? min(k, n) : n;
    double v;
    if (!map) {
      double dcg = 0.0, idcg = 0.0;
      for (int j = lane; j < kk; j += 32) { const double dj = discount(j); dcg += gain(ys[b + j], exp_gain) * dj; idcg += gain(ideal[b + j], exp_gain) * dj; }
      dcg = warp_sum(dcg); idcg = warp_sum(idcg);
      v = idcg == 0.0 ? (minus ? 0.0 : 1.0) : dcg / idcg;
    } else {                             // sum over the hits at r < k of hits(<= r) / (r + 1), over the relevant documents of the group
      int hits = 0; double acc = 0.0;
      for (int base = 0; base < n; base += 32) {
        const int j = base + lane;
        const bool rel = j < n && ys[b + j] > 0.0f;
        const unsigned bal = __ballot_sync(0xffffffffu, rel);
        const int h = hits + __popc(bal & (0xffffffffu >> (31 - lane)));
        if (rel && j < kk) acc += (double)h / (double)(j + 1);
        hits += __popc(bal);
      }
      acc = warp_sum(acc);
      v = hits == 0 ? (minus ? 0.0 : 1.0) : acc / (double)hits;
    }
    if (lane == 0) { const double wg = w ? (double)w[g] : 1.0; out[g] = wg * v; out[G + g] = wg; }
  }
}

// out[0] = sum of vals[0, G), out[1] = sum of vals[G, 2G), in a fixed order
__global__ void __launch_bounds__(kThreads) sum_pairs_kernel(const double* vals, int64_t G, double* out) {
  typedef cub::BlockReduce<double, kThreads> BR;
  __shared__ typename BR::TempStorage tmp;
  for (int half = 0; half < 2; ++half) {
    double v = 0.0;
    for (int64_t i = threadIdx.x; i < G; i += kThreads) v += vals[half * G + i];
    const double t = BR(tmp).Sum(v);
    if (threadIdx.x == 0) out[half] = t;
    __syncthreads();
  }
}

void rank_metric(const float* margin, const float* label, const float* weight, const RankGroups& rg, int map, int k, int exp_gain, int minus,
                 RankScratch* sc, double* out, cudaStream_t s) {
  B200_CHECK(rg.valid, "ranking metric: the query groups are not built");
  if (rg.n == 0) { CUDA_OK(cudaMemsetAsync(out, 0, 2 * sizeof(double), s)); return; }
  const int64_t G = rg.G;
  rank_sort(margin, label, rg, sc, s);
  sc->group.ensure(2 * (size_t)G);
  rank_metric_kernel<<<blocks_for(G * 32, kThreads), kThreads, 0, s>>>(sc->y_sorted.p, rg.ideal.p, rg.ptr.p, G, map, k, exp_gain, minus, weight, sc->group.p);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  sum_pairs_kernel<<<1, kThreads, 0, s>>>(sc->group.p, G, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
