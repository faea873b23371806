// curve.cu -- the curve pass of `aucpr` (binary and one-vs-rest) and of one-vs-rest `auc`: sort the scores of one class
// descending, walk the blocks of tied scores from the highest score down with running (positive, negative) weight sums,
// and add one ROC trapezoid or one PR segment per block.  DESIGN.md "AUC family" states the definitions; the double
// restatement is tests/auc_reference.py.
//
// Every sum runs in a fixed order over fixed tiles of kTile rows (no floating-point atomics): the running sums are a
// three-kernel scan (tile totals, one block scans the totals, each tile scans itself from its offset), the per-block
// terms are summed per tile and then by one block.  So the value is the same from run to run and for any grid size.
// Built with --fmad=false (build.py), so the terms round like the host restatement.  The scratch lives on the Booster
// (CurveScratch) and only grows; the K classes of a multi-class model reuse the same n-sized buffers one after another.
#include <cub/cub.cuh>
#include <cmath>
#include "curve.h"
#include "engine.h"

namespace b200 {

namespace {

constexpr int kThreads = 256, kRounds = 8, kTile = kThreads * kRounds;

struct Add2 {
  __device__ __forceinline__ double2 operator()(const double2& a, const double2& b) const { return make_double2(a.x + b.x, a.y + b.y); }
};
typedef cub::BlockScan<double2, kThreads> Scan2;
typedef cub::BlockReduce<double, kThreads> Reduce;

__host__ __device__ __forceinline__ int64_t tiles_for(int64_t n) { return (n + kTile - 1) / kTile; }
int grid_for_tiles(int64_t tiles) { return (int)std::max<int64_t>(1, std::min<int64_t>(tiles, (int64_t)engine_num_sms() * 8)); }

struct MassArgs {
  const int* order; const float* label; const float* weight; int64_t n;
  int K, c;                       // K == 0: binary (positive share = label); else positives are (int)label == c
};

// row at sorted position i: (w y, w (1 - y)); flags a binary label outside [0, 1]
__device__ __forceinline__ double2 row_mass(const MassArgs& a, int64_t i, unsigned* bad) {
  const int r = a.order[i];
  const double w = a.weight ? (double)a.weight[r] : 1.0;
  double y;
  if (a.K) y = (int)a.label[r] == a.c ? 1.0 : 0.0;
  else {
    const float l = a.label[r];
    if (!(l >= 0.0f && l <= 1.0f)) atomicOr(bad, 1u);
    y = (double)l;
  }
  return make_double2(w * y, w * (1.0 - y));
}

// pass 1: each row's mass into cum, each tile's total into tile (summed round by round, as pass 3 walks it)
__global__ void __launch_bounds__(kThreads) curve_mass_kernel(MassArgs a, double2* cum, double2* tile, unsigned* bad) {
  __shared__ typename Scan2::TempStorage tmp;
  const int64_t tiles = tiles_for(a.n);
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    double2 carry = make_double2(0.0, 0.0);
    for (int k = 0; k < kRounds; ++k) {
      const int64_t i = t * kTile + (int64_t)k * kThreads + threadIdx.x;
      const double2 v = i < a.n ? row_mass(a, i, bad) : make_double2(0.0, 0.0);
      if (i < a.n) cum[i] = v;
      double2 inc, agg;
      Scan2(tmp).InclusiveScan(v, inc, Add2(), agg);
      carry = Add2()(carry, agg);
      __syncthreads();
    }
    if (threadIdx.x == 0) tile[t] = carry;
  }
}

// pass 2 (one block): tile[t] = the sum of the tiles before t, in tile order
__global__ void __launch_bounds__(kThreads) curve_tile_offsets_kernel(double2* tile, int64_t tiles) {
  __shared__ typename Scan2::TempStorage tmp;
  double2 carry = make_double2(0.0, 0.0);
  for (int64_t b = 0; b < tiles; b += kThreads) {
    const int64_t j = b + threadIdx.x;
    const double2 v = j < tiles ? tile[j] : make_double2(0.0, 0.0);
    double2 ex, agg;
    Scan2(tmp).ExclusiveScan(v, ex, make_double2(0.0, 0.0), Add2(), agg);
    if (j < tiles) tile[j] = Add2()(carry, ex);
    carry = Add2()(carry, agg);
    __syncthreads();
  }
}

// pass 3: cum[i] = the running (tp, fp) through row i; end[i] = 1 where a block of tied scores ends
__global__ void __launch_bounds__(kThreads) curve_scan_kernel(double2* cum, const double2* tile, const float* key, int64_t n, unsigned char* end) {
  __shared__ typename Scan2::TempStorage tmp;
  const int64_t tiles = tiles_for(n);
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    double2 carry = tile[t];
    for (int k = 0; k < kRounds; ++k) {
      const int64_t i = t * kTile + (int64_t)k * kThreads + threadIdx.x;
      const double2 v = i < n ? cum[i] : make_double2(0.0, 0.0);
      double2 inc, agg;
      Scan2(tmp).InclusiveScan(v, inc, Add2(), agg);
      if (i < n) { cum[i] = Add2()(carry, inc); end[i] = (i == n - 1 || key[i] != key[i + 1]) ? 1 : 0; }
      carry = Add2()(carry, agg);
      __syncthreads();
    }
  }
}

// one block end j: its ROC trapezoid (unnormalised, as auc.cu) or its PR segment (Davis-Goadrich, in recall units)
__device__ __forceinline__ double block_term(const double2* ends, int64_t j, double P, int pr) {
  const double tp0 = j ? ends[j - 1].x : 0.0, fp0 = j ? ends[j - 1].y : 0.0, tp1 = ends[j].x, fp1 = ends[j].y;
  if (!pr) return (fp1 - fp0) * (tp1 + tp0) * 0.5;
  if (tp1 == tp0 || P <= 0.0) return 0.0;
  const double h = (fp1 - fp0) / (tp1 - tp0), a = 1.0 + h, b = (fp0 - h * tp0) / P;
  const double r0 = tp0 / P, r1 = tp1 / P;
  // ln(a r1 + b) - ln(a r0 + b) as log1p(a (r1 - r0) / (a r0 + b)): the difference of two logs loses their last bits, which
  // b / a (up to N / P on imbalanced data) would magnify; log1p keeps the segment's error within a few ulps of r1 - r0
  if (b != 0.0) return ((r1 - r0) - b / a * log1p(a * (r1 - r0) / (a * r0 + b))) / a;
  return (r1 - r0) / a;
}

// pass 4: part[t] = the sum of the terms of block ends [t kTile, (t + 1) kTile) (zero past the m ends)
__global__ void __launch_bounds__(kThreads) curve_area_kernel(const double2* ends, const int* m_ptr, int64_t tiles, int pr, double* part) {
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t m = *m_ptr;
  const double P = m ? ends[m - 1].x : 0.0;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    double acc = 0.0;
    for (int k = 0; k < kRounds; ++k) {
      const int64_t j = t * kTile + (int64_t)k * kThreads + threadIdx.x;
      if (j < m) acc += block_term(ends, j, P, pr);
    }
    const double s = Reduce(tmp).Sum(acc);
    if (threadIdx.x == 0) part[t] = s;
    __syncthreads();
  }
}

// pass 5 (one block): cls[3 c ..] = (area, P, N) of class c, the area summed over the tiles in a fixed order
__global__ void __launch_bounds__(kThreads) curve_class_kernel(const double* part, int64_t tiles, const double2* ends, const int* m_ptr, double* cls) {
  __shared__ typename Reduce::TempStorage tmp;
  double acc = 0.0;
  for (int64_t t = threadIdx.x; t < tiles; t += kThreads) acc += part[t];
  const double s = Reduce(tmp).Sum(acc);
  if (threadIdx.x == 0) {
    const int m = *m_ptr;
    cls[0] = s; cls[1] = m ? ends[m - 1].x : 0.0; cls[2] = m ? ends[m - 1].y : 0.0;
  }
}

// the classes into the per-rank vector: ROC (K >= 2) [area_c..., P_c N_c..., P_c...]; PR [value, P, N, bad], value the
// binary aucpr or the mean over classes, nan when a class has no positive or no negative weight
__global__ void curve_combine_kernel(const double* cls, int K, int pr, const unsigned* bad, double* vec) {
  if (!pr) {
    for (int c = 0; c < K; ++c) { const double* v = cls + 3 * c; vec[c] = v[0]; vec[K + c] = v[1] * v[2]; vec[2 * K + c] = v[1]; }
    return;
  }
  const int classes = K ? K : 1;
  double sum = 0.0;
  for (int c = 0; c < classes; ++c) { const double* v = cls + 3 * c; sum += (v[1] > 0.0 && v[2] > 0.0) ? v[0] : nan(""); }
  vec[0] = K ? sum / (double)K : sum;
  vec[1] = K ? 0.0 : cls[1]; vec[2] = K ? 0.0 : cls[2];
  vec[3] = *bad ? 1.0 : 0.0;
}

// out[0..3] from the all-reduced vector (header)
__global__ void curve_finish_kernel(const double* vec, int K, int pr, int world, double* out) {
  if (pr) { out[0] = vec[0] / (double)world; out[1] = vec[1]; out[2] = vec[2]; out[3] = vec[3]; return; }
  double num = 0.0, den = 0.0;
  bool degenerate = false;
  for (int c = 0; c < K; ++c) {
    if (vec[K + c] == 0.0) degenerate = true;
    else num += vec[c] / vec[K + c] * vec[2 * K + c];
    den += vec[2 * K + c];
  }
  out[0] = degenerate ? nan("") : num / den; out[1] = out[2] = out[3] = 0.0;
}

}  // namespace

int curve_metric_local(const float* margin, const float* label, const float* weight, int64_t n, int K, int logistic, int pr,
                       CurveScratch* sc, cudaStream_t s) {
  B200_CHECK(n < (int64_t)0x7fffffff, "aucpr / multi-class auc: too many rows");
  B200_CHECK(pr || K >= 2, "curve_metric_local: ROC is for one-vs-rest classes only");
  const int classes = K ? K : 1;
  const int64_t tiles = tiles_for(n);
  sc->cls.ensure(3 * (size_t)classes); sc->vec.ensure(std::max(3 * classes, 4)); sc->bad.ensure(1); sc->m.ensure(1);
  CUDA_OK(cudaMemsetAsync(sc->bad.p, 0, sizeof(unsigned), s));
  if (n == 0) CUDA_OK(cudaMemsetAsync(sc->cls.p, 0, 3 * classes * sizeof(double), s));
  else {
    sc->key.ensure(n); sc->key_sorted.ensure(n); sc->iota.ensure(n); sc->order.ensure(n); sc->cum.ensure(n); sc->ends.ensure(n);
    sc->end_flag.ensure(n); sc->tile.ensure(tiles); sc->part.ensure(tiles);
    size_t bytes = 0, need = 0;
    CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(nullptr, need, sc->key.p, sc->key_sorted.p, sc->iota.p, sc->order.p, (int)n, 0, 32, s));
    bytes = std::max(bytes, need);
    CUDA_OK(cub::DeviceSelect::Flagged(nullptr, need, sc->cum.p, sc->end_flag.p, sc->ends.p, sc->m.p, (int)n, s));
    bytes = std::max(bytes, need);
    sc->tmp.ensure(std::max<size_t>(bytes, 1));
    const int grid = grid_for_tiles(tiles);
    for (int c = 0; c < classes; ++c) {
      launch_curve_scores(margin, n, K, c, logistic, sc->key.p, sc->iota.p, s);
      size_t b = bytes;
      CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(sc->tmp.p, b, sc->key.p, sc->key_sorted.p, sc->iota.p, sc->order.p, (int)n, 0, 32, s));
      MassArgs ma{sc->order.p, label, weight, n, K, c};
      curve_mass_kernel<<<grid, kThreads, 0, s>>>(ma, sc->cum.p, sc->tile.p, sc->bad.p); ++g_kernel_launches;
      curve_tile_offsets_kernel<<<1, kThreads, 0, s>>>(sc->tile.p, tiles); ++g_kernel_launches;
      curve_scan_kernel<<<grid, kThreads, 0, s>>>(sc->cum.p, sc->tile.p, sc->key_sorted.p, n, sc->end_flag.p); ++g_kernel_launches;
      b = bytes;
      CUDA_OK(cub::DeviceSelect::Flagged(sc->tmp.p, b, sc->cum.p, sc->end_flag.p, sc->ends.p, sc->m.p, (int)n, s));
      curve_area_kernel<<<grid, kThreads, 0, s>>>(sc->ends.p, sc->m.p, tiles, pr, sc->part.p); ++g_kernel_launches;
      curve_class_kernel<<<1, kThreads, 0, s>>>(sc->part.p, tiles, sc->ends.p, sc->m.p, sc->cls.p + 3 * c); ++g_kernel_launches;
      CUDA_OK(cudaGetLastError());
    }
  }
  curve_combine_kernel<<<1, 1, 0, s>>>(sc->cls.p, K, pr, sc->bad.p, sc->vec.p); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  return pr ? 4 : 3 * K;
}

void curve_metric_finish(int K, int pr, int world, CurveScratch* sc, double* out, cudaStream_t s) {
  curve_finish_kernel<<<1, 1, 0, s>>>(sc->vec.p, K, pr, world, out); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}

}  // namespace b200
