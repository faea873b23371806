// ingest.cu -- training loaders that reach the device WITHOUT a dense float32 copy on the host (SURVEY.md section 8(f) row 2).
//   * columnar input (Parquet through pyarrow, pandas frames): the container's loader builds the matrix on the host two to
//     three times (data_utils.py:368-390: read_table -> to_pandas -> to_numpy -> data[:, 1:] -> DMatrix); here every column
//     buffer goes over PCIe as it is (float32 / float64 / int32 / int64 / uint8 / ..., at most 32 columns x kChunkRows at a
//     time through a staging buffer) and a tile kernel converts and transposes it into the engine's row-major float32 matrix.
//   * CSR input (libsvm channels, data_utils.py:348-365; scipy payloads, encoder.py:76-98): indptr / indices / values are
//     uploaded as they are and scattered into a NaN-filled matrix on the device (upstream keeps CSR; the hist path bins a dense
//     matrix anyway).
// Both are HBM / PCIe-bound byte movers: coalesced reads along the rows of one column, 128-byte row segments on the write side.
#include <algorithm>
#include <cmath>
#include <cstring>
#include "booster.h"
#include "comm.h"

namespace b200 {

namespace {
constexpr int kTileCols = 32;                 // columns per staged group == floats per written row segment (128 B)
constexpr int64_t kChunkRows = 1 << 22;       // rows per staged chunk: 32 columns x 4 Mi rows x 8 B = 1 GiB of staging at most

// column type codes of XGB200DMatrixCreateFromColumns (include/b200xgb.h)
enum ColType { kF32 = 0, kF64 = 1, kI32 = 2, kI64 = 3, kU8 = 4, kI8 = 5, kI16 = 6, kU16 = 7, kU32 = 8, kU64 = 9, kBool = 10 };
__host__ __device__ inline int col_itemsize(int t) {
  switch (t) { case kF32: case kI32: case kU32: return 4; case kF64: case kI64: case kU64: return 8; case kI16: case kU16: return 2; default: return 1; }
}
__device__ __forceinline__ float load_as_float(const unsigned char* p, int t, int64_t i) {
  switch (t) {                                 // round-to-nearest-even conversions, the ones numpy's astype(float32) performs
    case kF32: return reinterpret_cast<const float*>(p)[i];
    case kF64: return (float)reinterpret_cast<const double*>(p)[i];
    case kI32: return (float)reinterpret_cast<const int*>(p)[i];
    case kI64: return (float)reinterpret_cast<const long long*>(p)[i];
    case kU8: case kBool: return (float)p[i];
    case kI8: return (float)reinterpret_cast<const signed char*>(p)[i];
    case kI16: return (float)reinterpret_cast<const short*>(p)[i];
    case kU16: return (float)reinterpret_cast<const unsigned short*>(p)[i];
    case kU32: return (float)reinterpret_cast<const unsigned*>(p)[i];
    default: return (float)reinterpret_cast<const unsigned long long*>(p)[i];
  }
}

struct TileArgs {
  const unsigned char* col[kTileCols];        // staged column chunks (device)
  int type[kTileCols];
  int dst[kTileCols];                          // feature index in X, -1 = label, -2 = weight
  int ncols;
};

// One CTA = 32 rows x up to 32 columns: warp w reads column (w, w+8, ...) for 32 consecutive rows (coalesced), the tile goes
// through shared memory, and every row is written as one contiguous run of feature floats.
__global__ void __launch_bounds__(256) columns_to_rows_kernel(TileArgs a, int64_t rows, int64_t row0, int F, int f0, int nfeat,
                                                              float* __restrict__ X, float* __restrict__ y, float* __restrict__ w) {
  __shared__ float tile[kTileCols][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = (int64_t)blockIdx.x * 32; base < rows; base += (int64_t)gridDim.x * 32) {
    const int64_t r = base + lane;
    for (int c = warp; c < a.ncols; c += 8) {
      float v = 0.0f;
      if (r < rows) v = load_as_float(a.col[c], a.type[c], r);
      if (a.dst[c] >= 0) tile[a.dst[c] - f0][lane] = v;
      else if (r < rows) { if (a.dst[c] == -1) y[row0 + r] = v; else w[row0 + r] = v; }
    }
    __syncthreads();
    for (int rr = warp; rr < 32; rr += 8) {
      const int64_t row = base + rr;
      if (row < rows && lane < nfeat) X[(row0 + row) * F + f0 + lane] = tile[lane][rr];
    }
    __syncthreads();
  }
}

__global__ void fill_nan_kernel(float* X, int64_t count) {
  const float nan = __int_as_float(0x7fc00000);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) X[i] = nan;
}
// one warp per row: the row's entries land in its own F floats.  An index repeated inside a row keeps the value that comes
// last in the row: within a 32-entry chunk only the highest lane of each index stores, and chunks are ordered by __syncwarp.
__global__ void csr_scatter_kernel(const unsigned long long* __restrict__ indptr, const unsigned* __restrict__ indices, const float* __restrict__ vals,
                                   int64_t nrow, int F, float* __restrict__ X) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nrow; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const unsigned long long a = indptr[r], z = indptr[r + 1];
    for (unsigned long long j0 = a; j0 < z; j0 += 32) {
      const unsigned long long j = j0 + lane;
      const unsigned c = j < z ? indices[j] : 0xffffffffu;                      // F < 2^31: no real index equals the pad
      const unsigned same = __match_any_sync(0xffffffffu, c);
      if (j < z && (same >> lane) == 1u) X[r * F + c] = vals[j];
      __syncwarp();
    }
  }
}
}  // namespace

void csr_to_dense_device(const unsigned long long* d_ptr, const unsigned* d_idx, const float* d_val, int64_t nrow, int F, float* X, cudaStream_t s) {
  if (nrow * (int64_t)F <= 0) return;
  const int sms = engine_num_sms();
  fill_nan_kernel<<<sms * 8, 256, 0, s>>>(X, nrow * (int64_t)F); ++g_kernel_launches;
  const int grid = (int)std::min<int64_t>((nrow * 32 + 255) / 256, (int64_t)sms * 16);
  csr_scatter_kernel<<<std::max(grid, 1), 256, 0, s>>>(d_ptr, d_idx, d_val, nrow, F, X); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}

std::unique_ptr<DMatrix> DMatrix::from_columns(const void* const* cols, const int* types, int ncols, int64_t nrow, int label_col, int weight_col) {
  B200_CHECK(ncols >= 0 && nrow >= 0 && nrow < (int64_t)0x7fffffff, "DMatrix: bad shape");
  B200_CHECK(label_col < ncols && weight_col < ncols && (label_col < 0 || label_col != weight_col), "DMatrix: label / weight column out of range");
  for (int c = 0; c < ncols; ++c) { B200_CHECK(types[c] >= kF32 && types[c] <= kBool, "DMatrix: unknown column type code " + std::to_string(types[c])); B200_CHECK(cols[c] != nullptr || nrow == 0, "DMatrix: NULL column"); }
  auto dm = std::make_unique<DMatrix>();
  const int F = ncols - (label_col >= 0 ? 1 : 0) - (weight_col >= 0 ? 1 : 0);
  dm->n = nrow; dm->F = F;
  cudaStream_t s = engine_stream();
  dm->X.alloc((size_t)nrow * std::max(F, 0));
  DevBuf<float> dy, dw; dy.alloc(label_col >= 0 ? nrow : 0); dw.alloc(weight_col >= 0 ? nrow : 0);
  std::vector<int> dst(ncols); { int f = 0; for (int c = 0; c < ncols; ++c) dst[c] = c == label_col ? -1 : (c == weight_col ? -2 : f++); }
  const int64_t chunk = std::min<int64_t>(kChunkRows, std::max<int64_t>(nrow, 1));
  DevBuf<unsigned char> stage; stage.alloc((size_t)kTileCols * (size_t)chunk * 8);
  // groups: label / weight columns ride with the first group; feature columns in runs of <= 32 CONSECUTIVE feature indices
  std::vector<std::vector<int>> groups;
  { std::vector<int> cur; int feats = 0;
    for (int c = 0; c < ncols; ++c) { cur.push_back(c); if (dst[c] >= 0) ++feats; if (feats == kTileCols || (int)cur.size() == kTileCols) { groups.push_back(cur); cur.clear(); feats = 0; } }
    if (!cur.empty()) groups.push_back(cur); }
  for (int64_t row0 = 0; row0 < nrow; row0 += chunk) {
    const int64_t rows = std::min(chunk, nrow - row0);
    for (auto& g : groups) {
      TileArgs a{}; a.ncols = (int)g.size(); int f0 = -1, nfeat = 0;
      for (int k = 0; k < a.ncols; ++k) {
        const int c = g[k]; const int isz = col_itemsize(types[c]);
        unsigned char* d = stage.p + (size_t)k * (size_t)chunk * 8;
        CUDA_OK(cudaMemcpyAsync(d, (const unsigned char*)cols[c] + (size_t)row0 * isz, (size_t)rows * isz, cudaMemcpyHostToDevice, s));
        a.col[k] = d; a.type[k] = types[c]; a.dst[k] = dst[c];
        if (dst[c] >= 0) { if (f0 < 0) f0 = dst[c]; ++nfeat; }
      }
      if (f0 < 0) f0 = 0;
      const int grid = (int)std::min<int64_t>((rows + 31) / 32, (int64_t)engine_num_sms() * 8);
      columns_to_rows_kernel<<<std::max(grid, 1), 256, 0, s>>>(a, rows, row0, std::max(F, 1), f0, nfeat, dm->X.p, dy.p, dw.p); ++g_kernel_launches;
      CUDA_OK(cudaGetLastError());
    }
  }
  std::vector<float> hy(label_col >= 0 ? nrow : 0), hw(weight_col >= 0 ? nrow : 0);
  if (!hy.empty()) CUDA_OK(cudaMemcpyAsync(hy.data(), dy.p, sizeof(float) * nrow, cudaMemcpyDeviceToHost, s));
  if (!hw.empty()) CUDA_OK(cudaMemcpyAsync(hw.data(), dw.p, sizeof(float) * nrow, cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  dm->finish_upload(std::nanf(""));
  if (!hy.empty()) dm->set_float_info("label", hy.data(), hy.size());
  if (!hw.empty()) dm->set_float_info("weight", hw.data(), hw.size());
  return dm;
}

std::unique_ptr<DMatrix> DMatrix::from_csr(const size_t* indptr, const unsigned* indices, const float* data, size_t nindptr,
                                           size_t nelem, size_t ncol) {
  B200_CHECK(nindptr >= 1, "DMatrix: empty indptr");
  const size_t nrow = nindptr - 1;
  B200_CHECK(nrow < (size_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  B200_CHECK(indptr[nrow] <= nelem, "DMatrix: indptr runs past the end of the index / value arrays");
  size_t F = ncol;
  for (size_t i = 0; i < nelem; ++i) F = std::max<size_t>(F, (size_t)indices[i] + 1);
  for (size_t r = 0; r < nrow; ++r) B200_CHECK(indptr[r] <= indptr[r + 1], "DMatrix: indptr is not non-decreasing");
  auto dm = std::make_unique<DMatrix>();
  dm->n = (int64_t)nrow; dm->F = (int)F;
  cudaStream_t s = engine_stream();
  dm->X.alloc(nrow * F);
  if (nrow * F > 0) {
    static_assert(sizeof(size_t) == sizeof(unsigned long long), "indptr is uploaded as 64-bit offsets");
    DevBuf<unsigned long long> d_ptr; DevBuf<unsigned> d_idx; DevBuf<float> d_val;
    d_ptr.alloc(nindptr); d_idx.alloc(std::max<size_t>(nelem, 1)); d_val.alloc(std::max<size_t>(nelem, 1));
    CUDA_OK(cudaMemcpyAsync(d_ptr.p, indptr, sizeof(size_t) * nindptr, cudaMemcpyHostToDevice, s));
    if (nelem) { CUDA_OK(cudaMemcpyAsync(d_idx.p, indices, sizeof(unsigned) * nelem, cudaMemcpyHostToDevice, s));
                 CUDA_OK(cudaMemcpyAsync(d_val.p, data, sizeof(float) * nelem, cudaMemcpyHostToDevice, s)); }
    csr_to_dense_device(d_ptr.p, d_idx.p, d_val.p, (int64_t)nrow, (int)F, dm->X.p, s);
    Comm::get().sync_stream(s);                 // the staging buffers above die with this scope
  }
  dm->finish_upload(std::nanf(""));
  return dm;
}

}  // namespace b200
