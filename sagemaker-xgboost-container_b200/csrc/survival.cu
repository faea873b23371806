// survival.cu -- survival:aft (accelerated failure time on interval-censored labels) and survival:cox (Cox proportional
// hazards, Breslow ties): gradient pairs and the aft-nloglik / interval-regression-accuracy / cox-nloglik metrics.
// Formulas restate upstream xgboost src/common/survival_util.h, src/objective/aft_obj.cu, src/objective/regression_obj.cu
// (CoxRegression) and src/metric/survival_metric.cu, src/metric/elementwise_metric.cu (EvalCox) [UPSTREAM-RECALL].
// Compiled with --fmad=false (build.py): the double arithmetic rounds like a host restatement of the same expressions.
#include <cub/cub.cuh>
#include "survival.h"
#include "rng.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// AFT: the three distributions of z = (ln y - margin) / sigma [UPSTREAM-RECALL: survival_util.h]
// ---------------------------------------------------------------------------------------------
constexpr double kAftMinGrad = -15.0, kAftMaxGrad = 15.0, kAftMinHess = 1e-16, kAftMaxHess = 15.0, kAftEps = 1e-12;
enum Censor : int { kUncensored = 0, kRightCensored = 1, kLeftCensored = 2, kIntervalCensored = 3 };

__device__ __forceinline__ double aft_pdf(int d, double z) {
  if (d == kAftNormal) return exp(-z * z / 2.0) / sqrt(2.0 * 3.14159265358979323846);
  const double w = exp(z);
  if (d == kAftLogistic) { const double sd = 1.0 + w; return (isinf(w) || isinf(w * w)) ? 0.0 : w / (sd * sd); }
  return isinf(w) ? 0.0 : w * exp(-w);
}
__device__ __forceinline__ double aft_cdf(int d, double z) {
  if (d == kAftNormal) return 0.5 * (1.0 + erf(z / sqrt(2.0)));
  const double w = exp(z);
  if (d == kAftLogistic) return isinf(w) ? 1.0 : w / (1.0 + w);
  return 1.0 - exp(-w);
}
__device__ __forceinline__ double aft_grad_pdf(int d, double z) {
  if (d == kAftNormal) return -z * aft_pdf(d, z);
  const double w = exp(z);
  if (d == kAftLogistic) return isinf(w) ? 0.0 : aft_pdf(d, z) * (1.0 - w) / (1.0 + w);
  return isinf(w) ? 0.0 : (1.0 - w) * aft_pdf(d, z);
}
__device__ __forceinline__ double aft_hess_pdf(int d, double z) {
  if (d == kAftNormal) return (z * z - 1.0) * aft_pdf(d, z);
  const double w = exp(z);
  if (isinf(w) || isinf(w * w)) return 0.0;
  if (d == kAftLogistic) return aft_pdf(d, z) * (w * w - 4.0 * w + 1.0) / ((1.0 + w) * (1.0 + w));
  return (w * w - 3.0 * w + 1.0) * aft_pdf(d, z);
}

// the gradient / hessian where the prediction runs off to infinity, per distribution and censoring type; sign: z > 0 (for
// censored rows z_u > 0 || z_l > 0), i.e. the prediction sits below the label [UPSTREAM-RECALL: survival_util.h
// GetLimitGradAtInfPred / GetLimitHessAtInfPred]
__device__ __forceinline__ double aft_limit_grad(int d, int c, bool sign, double sigma) {
  if (d == kAftNormal) {
    switch (c) { case kUncensored: case kIntervalCensored: return sign ? kAftMinGrad : kAftMaxGrad;
                 case kRightCensored: return sign ? kAftMinGrad : 0.0; default: return sign ? 0.0 : kAftMaxGrad; }
  }
  if (d == kAftLogistic) {
    switch (c) { case kUncensored: case kIntervalCensored: return sign ? -1.0 / sigma : 1.0 / sigma;
                 case kRightCensored: return sign ? -1.0 / sigma : 0.0; default: return sign ? 0.0 : 1.0 / sigma; }
  }
  switch (c) { case kUncensored: case kIntervalCensored: return sign ? kAftMinGrad : 1.0 / sigma;
               case kRightCensored: return sign ? kAftMinGrad : 0.0; default: return sign ? 0.0 : 1.0 / sigma; }
}
__device__ __forceinline__ double aft_limit_hess(int d, int c, bool sign, double sigma) {
  if (d == kAftNormal) {
    switch (c) { case kUncensored: case kIntervalCensored: return 1.0 / (sigma * sigma);
                 case kRightCensored: return sign ? 1.0 / (sigma * sigma) : kAftMinHess; default: return sign ? kAftMinHess : 1.0 / (sigma * sigma); }
  }
  if (d == kAftLogistic) return kAftMinHess;
  switch (c) { case kLeftCensored: return kAftMinHess; default: return sign ? kAftMaxHess : kAftMinHess; }
}

__device__ __forceinline__ double clip(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }

// (g, h) of the AFT negative log-likelihood at margin m, clipped [UPSTREAM-RECALL: survival_util.h AFTLoss]
__device__ void aft_grad_hess(int d, double yl, double yu, double m, double sigma, double* g_out, double* h_out) {
  const double lyl = log(yl), lyu = log(yu);
  double gnum, gden, hnum, hden; int c; bool sign;
  if (yl == yu) {
    const double z = (lyl - m) / sigma;
    const double pdf = aft_pdf(d, z), gpdf = aft_grad_pdf(d, z), hpdf = aft_hess_pdf(d, z);
    c = kUncensored; sign = z > 0.0;
    gnum = gpdf; gden = sigma * pdf;
    hnum = -(pdf * hpdf - gpdf * gpdf); hden = sigma * sigma * pdf * pdf;
  } else {
    double zu = 0.0, zl = 0.0, pdf_u, pdf_l, cdf_u, cdf_l, gpdf_u, gpdf_l;
    c = kIntervalCensored;
    if (isinf(yu)) { pdf_u = 0.0; cdf_u = 1.0; gpdf_u = 0.0; c = kRightCensored; }
    else { zu = (lyu - m) / sigma; pdf_u = aft_pdf(d, zu); cdf_u = aft_cdf(d, zu); gpdf_u = aft_grad_pdf(d, zu); }
    if (yl <= 0.0) { pdf_l = 0.0; cdf_l = 0.0; gpdf_l = 0.0; c = kLeftCensored; }
    else { zl = (lyl - m) / sigma; pdf_l = aft_pdf(d, zl); cdf_l = aft_cdf(d, zl); gpdf_l = aft_grad_pdf(d, zl); }
    sign = zu > 0.0 || zl > 0.0;
    const double cdf_diff = cdf_u - cdf_l, pdf_diff = pdf_u - pdf_l, grad_diff = gpdf_u - gpdf_l;
    gnum = pdf_diff; gden = sigma * cdf_diff;
    hnum = -(cdf_diff * grad_diff - pdf_diff * pdf_diff);
    const double sd = sigma * cdf_diff; hden = sd * sd;
  }
  double g = gnum / gden, h = hnum / hden;
  if (gden < kAftEps && (isnan(g) || isinf(g))) g = aft_limit_grad(d, c, sign, sigma);
  if (hden < kAftEps && (isnan(h) || isinf(h))) h = aft_limit_hess(d, c, sign, sigma);
  *g_out = clip(g, kAftMinGrad, kAftMaxGrad); *h_out = clip(h, kAftMinHess, kAftMaxHess);
}

// negative log-likelihood of one row [UPSTREAM-RECALL: survival_util.h AFTLoss::Loss]
__device__ double aft_nloglik(int d, double yl, double yu, double m, double sigma) {
  if (yl == yu) {
    const double z = (log(yl) - m) / sigma;
    return -log(fmax(aft_pdf(d, z) / (sigma * yl), kAftEps));
  }
  const double cdf_u = isinf(yu) ? 1.0 : aft_cdf(d, (log(yu) - m) / sigma);
  const double cdf_l = yl <= 0.0 ? 0.0 : aft_cdf(d, (log(yl) - m) / sigma);
  return -log(fmax(cdf_u - cdf_l, kAftEps));
}

__device__ __forceinline__ void fold_absmax(float mg, float mh, unsigned* absmax) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
  __shared__ float sg[8], sh[8];
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
    if (absmax) { atomicMax(absmax, __float_as_uint(mg)); atomicMax(absmax + 1, __float_as_uint(mh)); }
  }
}

__device__ __forceinline__ bool row_dropped(const SurvivalGradArgs& a, int64_t r) {
  return a.subsample < 1.0f && !(rng_uniform(a.seed, 0x2000ull + a.iter, (unsigned long long)(r + a.row_offset)) < a.subsample);
}

__global__ void __launch_bounds__(256) aft_gradient_kernel(SurvivalGradArgs a) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    double g, h;
    aft_grad_hess(a.dist, (double)a.lower[r], (double)a.upper[r], (double)a.margin[r], (double)a.sigma, &g, &h);
    const float w = a.weight ? a.weight[r] : 1.0f;
    float gf = (float)g * w, hf = (float)h * w;
    if (row_dropped(a, r)) { gf = 0.f; hf = 0.f; }
    a.gpair[r] = make_float2(gf, hf);
    mg = fmaxf(mg, fabsf(gf)); mh = fmaxf(mh, hf);
  }
  fold_absmax(mg, mh, a.absmax);
}

__global__ void __launch_bounds__(256) aft_metric_kernel(const float* margin, const float* lower, const float* upper, const float* weight, int64_t n,
                                                         int dist, double sigma, int metric, double* out) {
  double s = 0, ws = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const double yl = lower[r], yu = upper[r], m = margin[r], w = weight ? (double)weight[r] : 1.0;
    double loss;
    if (metric == 0) loss = aft_nloglik(dist, yl, yu, m, sigma);
    else { const double p = exp(m); loss = (p >= yl && p <= yu) ? 1.0 : 0.0; }
    s += loss * w; ws += w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(out, s); atomicAdd(out + 1, ws); }
}

// ---------------------------------------------------------------------------------------------
// Deterministic scans: a fixed-order three-phase scan (per-tile sums, one CTA scans the tile sums in order, each tile scans
// itself with its carry).  No look-back and no atomics, so every sum depends only on the inputs and n.  Element j of the
// scan sits at position j (forward) or n - 1 - j (reverse: suffix sums).
// ---------------------------------------------------------------------------------------------
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems, kCarryThreads = 256;

__device__ __forceinline__ double add(double a, double b) { return a + b; }
__device__ __forceinline__ double2 add(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
template <class T> __device__ __forceinline__ T zero_of();
template <> __device__ __forceinline__ double zero_of<double>() { return 0.0; }
template <> __device__ __forceinline__ double2 zero_of<double2>() { return make_double2(0.0, 0.0); }
struct SumOp { template <class T> __device__ __forceinline__ T operator()(const T& a, const T& b) const { return add(a, b); } };

template <class T, bool REV, class Load>
__global__ void __launch_bounds__(kScanThreads) tile_sums_kernel(Load ld, int64_t n, T* tiles) {
  typedef cub::BlockReduce<T, kScanThreads> BR;
  __shared__ typename BR::TempStorage tmp;
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  T acc = zero_of<T>();
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t j = base + k * kScanThreads + threadIdx.x;
    if (j < n) acc = add(acc, ld(REV ? n - 1 - j : j));
  }
  const T tot = BR(tmp).Reduce(acc, SumOp());
  if (threadIdx.x == 0) tiles[blockIdx.x] = tot;
}

// in place: tiles[t] <- tiles[0] + ... + tiles[t - 1], and tiles[ntiles] <- the total
template <class T>
__global__ void __launch_bounds__(kCarryThreads) tile_carries_kernel(T* tiles, int64_t ntiles) {
  typedef cub::BlockScan<T, kCarryThreads> BS;
  __shared__ typename BS::TempStorage tmp;
  const int64_t per = (ntiles + kCarryThreads - 1) / kCarryThreads;
  const int64_t b = min((int64_t)threadIdx.x * per, ntiles), e = min(b + per, ntiles);
  T s = zero_of<T>();
  for (int64_t i = b; i < e; ++i) s = add(s, tiles[i]);
  T excl, total;
  BS(tmp).ExclusiveScan(s, excl, zero_of<T>(), SumOp(), total);
  for (int64_t i = b; i < e; ++i) { const T v = tiles[i]; tiles[i] = excl; excl = add(excl, v); }
  if (threadIdx.x == 0) tiles[ntiles] = total;
}

template <class T, bool REV, class Load>
__global__ void __launch_bounds__(kScanThreads) tile_scan_kernel(Load ld, int64_t n, const T* carries, T* out) {
  typedef cub::BlockExchange<T, kScanThreads, kScanItems> BX;
  typedef cub::BlockScan<T, kScanThreads> BS;
  __shared__ union { typename BX::TempStorage x; typename BS::TempStorage s; } tmp;
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  T v[kScanItems];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t j = base + k * kScanThreads + threadIdx.x;
    v[k] = j < n ? ld(REV ? n - 1 - j : j) : zero_of<T>();
  }
  BX(tmp.x).StripedToBlocked(v);
  __syncthreads();
  BS(tmp.s).InclusiveScan(v, v, SumOp());
  __syncthreads();
  const T c = carries[blockIdx.x];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) v[k] = add(c, v[k]);
  BX(tmp.x).BlockedToStriped(v);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t j = base + k * kScanThreads + threadIdx.x;
    if (j < n) out[REV ? n - 1 - j : j] = v[k];
  }
}

static int64_t num_tiles(int64_t n) { return (n + kScanTile - 1) / kScanTile; }

// tiles: num_tiles(n) + 1 entries; out: the inclusive scan (nullptr: only the total, left in tiles[num_tiles(n)])
template <class T, bool REV, class Load>
static void fixed_order_scan(Load ld, int64_t n, T* tiles, T* out, cudaStream_t s) {
  const int64_t nt = num_tiles(n);
  tile_sums_kernel<T, REV, Load><<<(unsigned)nt, kScanThreads, 0, s>>>(ld, n, tiles); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  tile_carries_kernel<T><<<1, kCarryThreads, 0, s>>>(tiles, nt); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  if (out) { tile_scan_kernel<T, REV, Load><<<(unsigned)nt, kScanThreads, 0, s>>>(ld, n, tiles, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
}

// ---------------------------------------------------------------------------------------------
// Cox (Breslow ties) [UPSTREAM-RECALL: regression_obj.cu CoxRegression::GetGradient].  In sorted order (stable, ascending |y|):
//   D_i = sum of exp(m_j) over the rows with |y_j| >= |y_i|   (a suffix sum taken from the tie-group head of i)
//   R_i = sum of 1 / D_k, S_i = sum of 1 / D_k^2 over the events at sorted positions <= i
//   g = (e_i R_i - [y_i > 0]) w_i,  h = (e_i R_i - e_i^2 S_i) w_i
// Upstream takes D as the total minus running prefixes; the suffix sum is the same quantity without the cancellation at the
// tail, so the two differ at rounding level (DESIGN.md).
// ---------------------------------------------------------------------------------------------
struct LoadValue { const double* v; __device__ __forceinline__ double operator()(int64_t i) const { return v[i]; } };
struct LoadInvD {                      // events: (1 / D, 1 / D^2), others (0, 0)
  const double* suffix; const int* head; const unsigned char* event;
  __device__ __forceinline__ double2 operator()(int64_t i) const {
    if (!event[i]) return make_double2(0.0, 0.0);
    const double d = suffix[head[i]];
    return make_double2(1.0 / d, 1.0 / (d * d));
  }
};
struct LoadNll {                       // events: (ln D - m, 1), others (0, 0)
  const float* margin; const int* order; const double* suffix; const int* head; const unsigned char* event;
  __device__ __forceinline__ double2 operator()(int64_t i) const {
    if (!event[i]) return make_double2(0.0, 0.0);
    return make_double2(log(suffix[head[i]]) - (double)margin[order[i]], 1.0);
  }
};

__global__ void __launch_bounds__(256) abs_iota_kernel(const float* y, int64_t n, float* key, int* idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) { key[i] = fabsf(y[i]); idx[i] = (int)i; }
}
__global__ void __launch_bounds__(256) tie_heads_kernel(const float* key, const int* order, const float* y, int64_t n, int* head, unsigned char* event) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    head[i] = (i == 0 || key[i] != key[i - 1]) ? (int)i : 0;
    event[i] = y[order[i]] > 0.0f ? 1 : 0;
  }
}
struct MaxInt { __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; } };

__global__ void __launch_bounds__(256) cox_exp_kernel(const float* margin, const int* order, int64_t n, double* e) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) e[i] = exp((double)margin[order[i]]);
}

__global__ void __launch_bounds__(256) cox_gradient_kernel(SurvivalGradArgs a, const int* order, const unsigned char* event, const double* e, const double2* rs) {
  float mg = 0.f, mh = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = order[i];
    const double ei = e[i]; const double2 q = rs[i];
    const double g = ei * q.x - (event[i] ? 1.0 : 0.0);
    const double h = ei * q.x - ei * ei * q.y;
    const double w = a.weight ? (double)a.weight[r] : 1.0;
    float gf = (float)(g * w), hf = (float)(h * w);
    if (row_dropped(a, r)) { gf = 0.f; hf = 0.f; }
    a.gpair[r] = make_float2(gf, hf);
    mg = fmaxf(mg, fabsf(gf)); mh = fmaxf(mh, hf);
  }
  fold_absmax(mg, mh, a.absmax);
}

// ---------------------------------------------------------------------------------------------
static inline int grid_for(int64_t n) { int64_t g = (n + 255) / 256; if (g < 1) g = 1; if (g > engine_num_sms() * 8) g = engine_num_sms() * 8; return (int)g; }

void CoxScratch::ensure(int64_t n) {
  e.ensure((size_t)n); suffix.ensure((size_t)n); rs.ensure((size_t)n); tiles.ensure((size_t)num_tiles(n) + 1);
}

void launch_aft_gradient(const SurvivalGradArgs& a, cudaStream_t s) {
  if (a.n == 0) return;
  aft_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

void launch_aft_metric(const float* margin, const float* lower, const float* upper, const float* weight, int64_t n, int dist, float sigma,
                       int metric, double* out, cudaStream_t s) {
  if (n == 0) return;
  aft_metric_kernel<<<grid_for(n), 256, 0, s>>>(margin, lower, upper, weight, n, dist, (double)sigma, metric, out); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}

void cox_sort(const float* label, int64_t n, CoxOrder* o, CoxScratch* sc, cudaStream_t s) {
  B200_CHECK(n < (int64_t)0x7fffffff, "survival:cox: more than 2^31-1 rows");
  o->order.alloc((size_t)n); o->head.alloc((size_t)n); o->event.alloc((size_t)n); o->n = n; o->valid = true;
  if (n == 0) return;
  DevBuf<float> key_in, key_out; DevBuf<int> idx_in; key_in.alloc((size_t)n); key_out.alloc((size_t)n); idx_in.alloc((size_t)n);
  abs_iota_kernel<<<grid_for(n), 256, 0, s>>>(label, n, key_in.p, idx_in.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  // radix sort is stable: ties keep row order
  size_t bytes = 0;
  CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, key_in.p, key_out.p, idx_in.p, o->order.p, (int)n, 0, 32, s));
  sc->tmp.ensure(bytes);
  CUDA_OK(cub::DeviceRadixSort::SortPairs(sc->tmp.p, bytes, key_in.p, key_out.p, idx_in.p, o->order.p, (int)n, 0, 32, s)); ++g_kernel_launches;
  tie_heads_kernel<<<grid_for(n), 256, 0, s>>>(key_out.p, o->order.p, label, n, idx_in.p, o->event.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  // head of each position: running max of the group starts (integer max: any scan order gives the same result)
  bytes = 0;
  CUDA_OK(cub::DeviceScan::InclusiveScan(nullptr, bytes, idx_in.p, o->head.p, MaxInt(), (int)n, s));
  sc->tmp.ensure(bytes);
  CUDA_OK(cub::DeviceScan::InclusiveScan(sc->tmp.p, bytes, idx_in.p, o->head.p, MaxInt(), (int)n, s)); ++g_kernel_launches;
  CUDA_OK(cudaStreamSynchronize(s));       // the key / index buffers are released on return
}

// e = exp(m) in sorted order and its suffix sums
static void cox_suffix(const float* margin, const CoxOrder& o, CoxScratch* sc, cudaStream_t s) {
  const int64_t n = o.n;
  sc->ensure(n);
  cox_exp_kernel<<<grid_for(n), 256, 0, s>>>(margin, o.order.p, n, sc->e.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  fixed_order_scan<double, true>(LoadValue{sc->e.p}, n, reinterpret_cast<double*>(sc->tiles.p), sc->suffix.p, s);
}

void launch_cox_gradient(const SurvivalGradArgs& a, const CoxOrder& o, CoxScratch* sc, cudaStream_t s) {
  if (a.n == 0) return;
  B200_CHECK(o.valid && o.n == a.n, "survival:cox: the label order does not match the matrix");
  cox_suffix(a.margin, o, sc, s);
  fixed_order_scan<double2, false>(LoadInvD{sc->suffix.p, o.head.p, o.event.p}, a.n, sc->tiles.p, sc->rs.p, s);
  cox_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a, o.order.p, o.event.p, sc->e.p, sc->rs.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

void cox_nloglik(const float* margin, int64_t n, const CoxOrder& o, CoxScratch* sc, double* out, cudaStream_t s) {
  if (n == 0) { CUDA_OK(cudaMemsetAsync(out, 0, 2 * sizeof(double), s)); return; }
  B200_CHECK(o.valid && o.n == n, "cox-nloglik: the label order does not match the matrix");
  cox_suffix(margin, o, sc, s);
  fixed_order_scan<double2, false>(LoadNll{margin, o.order.p, sc->suffix.p, o.head.p, o.event.p}, n, sc->tiles.p, (double2*)nullptr, s);
  CUDA_OK(cudaMemcpyAsync(out, sc->tiles.p + num_tiles(n), 2 * sizeof(double), cudaMemcpyDeviceToDevice, s));
}

}  // namespace b200
