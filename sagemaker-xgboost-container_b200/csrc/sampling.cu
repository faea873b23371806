// sampling.cu -- sampling_method=gradient_based (sampling.h): the threshold select and the sampling kernel.
//
// The threshold u of a column solves sum_i min(1, rag_i / u) = k.  phi(v) = sum_i min(rag_i, v) - k v is positive exactly for
// 0 < v < u, so u is found by a radix descent over the bits of rag (non-negative floats order as their uint32 bits): each
// pass builds one histogram of row counts and exact int64 fixed-point rag sums over the current bucket range, evaluates phi at
// every bucket's lower edge from the prefix counts and sums, and descends into the last bucket where phi > 0.  After the last
// pass that bucket is one value x with x < u <= next(x), and u = S_below / (k - #above) over the rows <= x and > x.
// Each bucket sums on its own grid, 2^(bits - e) for values below 2^e (a bucket of the first pass spans two binades), so a
// row keeps bits of precision next to rows many binades larger; the pick kernel adds the buckets' sums in double, in bucket
// order.  Integer sums and one fixed order of double operations: the result depends on the pairs alone, not on timing.
#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>
#include <algorithm>
#include "sampling.h"
#include "rng.h"

namespace b200 {
namespace cg = cooperative_groups;

static inline unsigned blocks_per_column(int64_t n, int K) {
  const int64_t want = (n + 255) / 256, cap = std::max<int64_t>(1, (int64_t)engine_num_sms() * 8 / std::max(K, 1));
  return (unsigned)std::max<int64_t>(1, std::min(want, cap));
}

// sqrtf(g^2 + lambda h^2), every operation rounded on its own (no fused multiply-add), as the NumPy restatement computes it
__device__ __forceinline__ float gbs_rag(float2 v) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(kGbsLambda, __fmul_rn(v.y, v.y))));
}
// the descent's key: the bits of a finite rag, non-finite rag (inf, NaN) at the bits of +inf, above every finite value
__device__ __forceinline__ unsigned gbs_key(float x) { return isfinite(x) ? __float_as_uint(x) : 0x7f800000u; }
// The grid of the bucket of keys [lo, lo + 2^shift): rag_q = rint(rag * 2^(bits - e)) <= 2^bits, every value of the bucket
// below 2^e (e from its largest key; 128 where the bucket reaches the non-finite keys), capped at 2^126 for denormal buckets.
__device__ __forceinline__ int gbs_grid_exp(unsigned lo, int shift, int bits) {
  const unsigned long long top = (unsigned long long)lo + (1ull << shift) - 1ull;
  int e = 128;
  if (top < 0x7f800000ull) { const float m = __uint_as_float((unsigned)top); e = 0; if (m > 0.f) frexpf(m, &e); }
  return min(bits - e, 126);
}

__global__ void __launch_bounds__(256) gbs_rag_kernel(const float2* gpair, int64_t gp_stride, int64_t n, float* rag) {
  const int k = blockIdx.y;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
    rag[(int64_t)k * gp_stride + r] = gbs_rag(gpair[(int64_t)k * gp_stride + r]);
}

// One pass: the rows whose key matches the column's prefix above this pass's digit add 1 and rag_q to their digit.  Rows
// of a warp that share a digit are combined first (many rows share the leading digits of their magnitude).
__global__ void __launch_bounds__(256) gbs_hist_kernel(const float* rag, int64_t gp_stride, int64_t n, const GbsState* st, unsigned long long* hist,
                                                       int pass, int bits) {
  const int k = blockIdx.y;
  const int shift = 32 - kGbsDigitBits * (pass + 1);
  const unsigned hi_mask = pass == 0 ? 0u : ~0u << (shift + kGbsDigitBits);
  const unsigned prefix = st[k].prefix;
  __shared__ unsigned long long cnt[kGbsBuckets], sum[kGbsBuckets];
  __shared__ float scale[kGbsBuckets];
  for (int b = threadIdx.x; b < kGbsBuckets; b += blockDim.x) {
    cnt[b] = 0; sum[b] = 0; scale[b] = ldexpf(1.0f, gbs_grid_exp(prefix | ((unsigned)b << shift), shift, bits));
  }
  __syncthreads();
  const cg::thread_block_tile<32> warp = cg::tiled_partition<32>(cg::this_thread_block());
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += (int64_t)gridDim.x * blockDim.x) {   // uniform per warp
    const int64_t r = base + threadIdx.x;
    unsigned digit = kGbsBuckets;            // no bucket
    unsigned long long q = 0;
    if (r < n) {
      const float x = rag[(int64_t)k * gp_stride + r];
      const unsigned key = gbs_key(x);
      if ((key & hi_mask) == prefix) {
        digit = (key >> shift) & (kGbsBuckets - 1);
        if (isfinite(x)) q = (unsigned long long)__float2ll_rn(__fmul_rn(x, scale[digit]));
      }
    }
    const cg::coalesced_group grp = cg::labeled_partition(warp, digit);
    const unsigned long long s = cg::reduce(grp, q, cg::plus<unsigned long long>());
    if (grp.thread_rank() == 0 && digit < (unsigned)kGbsBuckets) {
      atomicAdd(&cnt[digit], (unsigned long long)grp.size());
      if (s) atomicAdd(&sum[digit], s);
    }
  }
  __syncthreads();
  unsigned long long* h = hist + (size_t)k * 2 * kGbsBuckets;
  for (int b = threadIdx.x; b < kGbsBuckets; b += blockDim.x) {
    if (cnt[b]) atomicAdd(h + b, cnt[b]);
    if (sum[b]) atomicAdd(h + kGbsBuckets + b, sum[b]);
  }
}

// After pass `pass`, one thread per column: phi at every bucket's lower edge v (finite edges only), in double in this order:
// S_lt + v * (N_ge - k), S_lt accumulating each bucket's sum times 2^-(its grid exponent); the last edge with phi > 0 names the
// bucket to descend into (bucket 0 when none).
__global__ void gbs_pick_kernel(GbsState* st, const unsigned long long* hist, int K, long long k_target, int pass, int bits) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  GbsState g = st[k];
  const unsigned long long* hc = hist + (size_t)k * 2 * kGbsBuckets;
  const unsigned long long* hs = hc + kGbsBuckets;
  const int shift = 32 - kGbsDigitBits * (pass + 1);
  long long total = 0;
  for (int b = 0; b < kGbsBuckets; ++b) total += (long long)hc[b];
  int pick = 0;
  double s_lt = g.s_lo, s_pick = g.s_lo;
  long long n_ge = g.n_hi + total, n_pick = g.n_hi + total;
  for (int b = 0; b < kGbsBuckets; ++b) {
    const unsigned edge = g.prefix | ((unsigned)b << shift);
    if (edge >= 0x7f800000u) break;
    const double phi = __dadd_rn(s_lt, __dmul_rn((double)__uint_as_float(edge), (double)(n_ge - k_target)));
    if (phi > 0.0) { pick = b; s_pick = s_lt; n_pick = n_ge; }
    s_lt = __dadd_rn(s_lt, ldexp((double)hs[b], -gbs_grid_exp(edge, shift, bits))); n_ge -= (long long)hc[b];
  }
  const double s_bucket = ldexp((double)hs[pick], -gbs_grid_exp(g.prefix | ((unsigned)pick << shift), shift, bits));
  g.prefix |= (unsigned)pick << shift;
  g.s_lo = s_pick; g.n_hi = n_pick - (long long)hc[pick];         // rows below / above the chosen bucket
  if (pass == kGbsPasses - 1) {                                    // the bucket is the single value x = prefix
    const unsigned x = g.prefix;
    const double s_below = __dadd_rn(g.s_lo, s_bucket);
    const long long den = k_target - g.n_hi;
    float u = 0.f;                                                 // x == 0: no positive v has phi > 0, every row is kept
    if (x != 0u) u = s_below > 0.0 && den > 0 ? __double2float_rn(__ddiv_rn(s_below, (double)den)) : __uint_as_float(x + 1u);
    g.u = u;
  }
  st[k] = g;
}

void gradient_based_threshold(const float2* gpair, int64_t gp_stride, int64_t n, int K, float subsample, GbsScratch* sc, cudaStream_t s) {
  sc->rag.ensure((size_t)std::max<int64_t>(gp_stride, 1) * K); sc->hist.ensure((size_t)K * 2 * kGbsBuckets); sc->st.ensure((size_t)K);
  const long long k_target = gbs_target(n, subsample);
  const int bits = grad_bits_for(n);
  const dim3 grid(blocks_per_column(n, K), (unsigned)K);
  CUDA_OK(cudaMemsetAsync(sc->st.p, 0, sizeof(GbsState) * K, s));
  gbs_rag_kernel<<<grid, 256, 0, s>>>(gpair, gp_stride, n, sc->rag.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  for (int pass = 0; pass < kGbsPasses; ++pass) {
    CUDA_OK(cudaMemsetAsync(sc->hist.p, 0, sizeof(unsigned long long) * K * 2 * kGbsBuckets, s));
    gbs_hist_kernel<<<grid, 256, 0, s>>>(sc->rag.p, gp_stride, n, sc->st.p, sc->hist.p, pass, bits); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    gbs_pick_kernel<<<(K + 31) / 32, 32, 0, s>>>(sc->st.p, sc->hist.p, K, k_target, pass, bits); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  }
}

// p = rag / u.  u == 0: every row as it is; non-finite rag: kept as it is (p = 1); p >= 1: kept as it is; else kept with
// probability p as (g / p, h / p), zeroed otherwise (a zero pair has p = 0 and stays zero).  Since rag >= |g| and
// rag >= sqrt(lambda) h, a scaled pair has |g / p| <= u and h / p <= u / sqrt(lambda) up to rounding: the scales that
// absmax feeds stay finite.
__global__ void __launch_bounds__(256) gbs_sample_kernel(GbsSampleArgs a) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float draw = rng_uniform(a.seed, a.stream, (unsigned long long)(r + a.row_offset));
    for (int k = 0; k < a.K; ++k) {
      const float2 v = a.src[(int64_t)k * a.gp_stride + r];
      const float u = a.st[k].u;
      float2 o = v;
      if (u > 0.f) {
        const float x = gbs_rag(v);
        if (isfinite(x)) {
          const float p = __fdiv_rn(x, u);
          if (p < 1.f) o = draw < p ? make_float2(__fdiv_rn(v.x, p), __fdiv_rn(v.y, p)) : make_float2(0.f, 0.f);
        }
      }
      a.dst[(int64_t)k * a.gp_stride + r] = o;
      mg = fmaxf(mg, fabsf(o.x)); mh = fmaxf(mh, o.y);
    }
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

void launch_gradient_based_sample(const GbsSampleArgs& a, cudaStream_t s) {
  gbs_sample_kernel<<<blocks_per_column(a.n, 1), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
