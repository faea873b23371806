// inplace.h -- in-place prediction (Booster::inplace_predict, DESIGN.md "In-place prediction"): the caller's array described
// as it lies in memory, the typestr it is read as, and the row chunks a host array crosses PCIe in.  The host half needs no
// CUDA (tests/helpers/inplace_sweep.cc compiles it with g++); the device half is the loader the predictor kernels read through.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

namespace b200 {

// element types of an in-place input.  float32, float64 and float16 are read by the predictor kernels themselves; the others
// are converted tile by tile into a float32 scratch first (launch_convert_rows).
enum InType : int { kInF32 = 0, kInF64, kInF16, kInI8, kInI16, kInI32, kInI64, kInU8, kInU16, kInU32, kInU64, kInBool };

inline int in_itemsize(int t) {
  switch (t) { case kInF64: case kInI64: case kInU64: return 8; case kInF32: case kInI32: case kInU32: return 4;
               case kInF16: case kInI16: case kInU16: return 2; default: return 1; }
}
inline bool in_read_in_place(int t) { return t == kInF32 || t == kInF64 || t == kInF16; }

// numpy / __cuda_array_interface__ typestr -> InType; -1 with *why naming the cause for anything else (complex, object,
// datetime, big-endian, ...)
inline int in_type_of(const std::string& ts, std::string* why) {
  static const char* const names[] = {"<f4", "<f8", "<f2", "|i1", "<i2", "<i4", "<i8", "|u1", "<u2", "<u4", "<u8", "|b1"};
  for (int t = 0; t < 12; ++t) if (ts == names[t]) return t;
  const char k = ts.size() >= 2 ? ts[1] : '?';
  if (k == 'c') *why = "complex values (typestr " + ts + ") are not supported";
  else if (k == 'O') *why = "an object array (typestr " + ts + ") is not supported: convert it to a numeric dtype";
  else if (k == 'M' || k == 'm') *why = "datetime / timedelta values (typestr " + ts + ") are not supported";
  else if (!ts.empty() && ts[0] == '>') *why = "big-endian data (typestr " + ts + ") is not supported";
  else *why = "unsupported typestr " + ts;
  return -1;
}

// The caller's matrix: element (r, f) at ptr + r * s0 + f * s1 bytes (either stride may be the contiguous one, or negative),
// NaN or a value equal to `missing` (after the conversion to float32) is missing.  CSR: row r holds the float32 values at
// ptr[j] for j in [indptr[r], indptr[r + 1]) at columns indices[j]; absent entries are missing, `missing` does not apply, a
// column repeated inside a row keeps its last value.
struct InputDesc {
  const void* ptr = nullptr; int type = kInF32;
  int64_t s0 = 0, s1 = 0;
  int64_t n = 0; int F = 0;
  float missing = __builtin_nanf("");
  const int64_t* indptr = nullptr; const int32_t* indices = nullptr;     // CSR when indptr != nullptr
};

// Staging of host inputs: two buffers of kInplaceStageBytes (pinned on the host, device memory on the Booster), whatever n is.
constexpr size_t kInplaceStageBytes = size_t(32) << 20;

// rows per chunk of a host dense array with row_bytes bytes per row (its own dtype) through buffers of cap bytes; debug_rows > 0
// caps the rows further (a debug knob that lets a small array span several chunks).  At least one row per chunk: rows wider
// than the cap are refused by the caller (inplace_row_fits).
inline int64_t inplace_chunk_rows(int64_t n, int64_t row_bytes, size_t cap, int64_t debug_rows) {
  int64_t rows = row_bytes > 0 ? (int64_t)(cap / (size_t)row_bytes) : n;
  if (debug_rows > 0 && debug_rows < rows) rows = debug_rows;
  if (rows > n) rows = n;
  return rows < 1 ? 1 : rows;
}
inline bool inplace_row_fits(int64_t row_bytes, size_t cap) { return row_bytes >= 0 && (size_t)row_bytes <= cap; }

// bytes of CSR rows [r0, r1) in the staging buffer: their r1 - r0 + 1 offsets (int64), then indices (int32) and values
// (float32) of their entries, each part 16 B aligned
inline size_t inplace_csr_bytes(int64_t rows, int64_t nnz) {
  auto al = [](size_t b) { return (b + 15) & ~size_t(15); };
  return al((size_t)(rows + 1) * 8) + al((size_t)nnz * 4) * 2;
}
// the end of the CSR chunk that starts at row r0: as many rows as fit the cap (and debug_rows), at least one; returns r0 when
// row r0 alone does not fit
inline int64_t inplace_csr_chunk_end(const int64_t* indptr, int64_t n, int64_t r0, size_t cap, int64_t debug_rows) {
  int64_t lo = r0, hi = n;
  if (debug_rows > 0 && r0 + debug_rows < hi) hi = r0 + debug_rows;
  if (inplace_csr_bytes(1, indptr[r0 + 1] - indptr[r0]) > cap) return r0;
  while (lo < hi) {                                    // the largest end in (r0, hi] that fits: the bytes grow with the end
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if (inplace_csr_bytes(mid - r0, indptr[mid] - indptr[r0]) <= cap) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace b200

#ifdef __CUDACC__
#include <cuda_fp16.h>
namespace b200 {

// element (r, f) of a dense input as float32, rounded to nearest even, NaN when missing
template <int T>
__device__ __forceinline__ float in_load(const unsigned char* p) {
  if (T == kInF32) return __ldg(reinterpret_cast<const float*>(p));
  if (T == kInF64) return __double2float_rn(__ldg(reinterpret_cast<const double*>(p)));
  if (T == kInF16) return __half2float(__ldg(reinterpret_cast<const __half*>(p)));
  if (T == kInI8) return __int2float_rn(*reinterpret_cast<const signed char*>(p));
  if (T == kInI16) return __int2float_rn(*reinterpret_cast<const short*>(p));
  if (T == kInI32) return __int2float_rn(__ldg(reinterpret_cast<const int*>(p)));
  if (T == kInI64) return __ll2float_rn(__ldg(reinterpret_cast<const long long*>(p)));
  if (T == kInU8 || T == kInBool) return __uint2float_rn(*p);
  if (T == kInU16) return __uint2float_rn(*reinterpret_cast<const unsigned short*>(p));
  if (T == kInU32) return __uint2float_rn(__ldg(reinterpret_cast<const unsigned*>(p)));
  return __ull2float_rn(__ldg(reinterpret_cast<const unsigned long long*>(p)));
}
template <int T>
__device__ __forceinline__ float load_x(const InputDesc& d, int64_t r, int f) {
  const float v = in_load<T>(static_cast<const unsigned char*>(d.ptr) + r * d.s0 + (int64_t)f * d.s1);
  return v == d.missing ? __int_as_float(0x7fc00000) : v;
}
// the runtime-typed loader (the conversion into the float32 scratch)
__device__ __forceinline__ float load_x(const InputDesc& d, int64_t r, int f) {
  switch (d.type) {
    case kInF32: return load_x<kInF32>(d, r, f); case kInF64: return load_x<kInF64>(d, r, f); case kInF16: return load_x<kInF16>(d, r, f);
    case kInI8: return load_x<kInI8>(d, r, f); case kInI16: return load_x<kInI16>(d, r, f); case kInI32: return load_x<kInI32>(d, r, f);
    case kInI64: return load_x<kInI64>(d, r, f); case kInU8: return load_x<kInU8>(d, r, f); case kInU16: return load_x<kInU16>(d, r, f);
    case kInU32: return load_x<kInU32>(d, r, f); case kInU64: return load_x<kInU64>(d, r, f); default: return load_x<kInBool>(d, r, f);
  }
}

// Sources of the predictor kernels (misc.cu, dart.cu): stage() fills a tile of `rows` rows from row r0 into shared memory
// (pitch floats per row, the caller synchronises around it); at() is one element for the thread-per-row walks, NaN for a
// feature the matrix lacks.
// The DMatrix's float32 matrix (row-major, NaN = missing): predict()'s own path.
struct RowsF32 {
  const float* X; int F;
  __device__ __forceinline__ void stage(float* s_x, int pitch, int64_t r0, int rows) const {
    const float* src = X + r0 * F;
    const int total = rows * F;
    for (int i = threadIdx.x; i < total; i += blockDim.x) { const int r = i / F, f = i - r * F; s_x[r * pitch + f] = __ldg(src + i); }
  }
  __device__ __forceinline__ float at(int64_t r, int f) const { return f < F ? __ldg(X + r * F + f) : __int_as_float(0x7fc00000); }
};
// A strided dense input of element type T: threads run along whichever of rows and columns is contiguous in memory.
template <int T>
struct StridedSrc {
  InputDesc d;
  __device__ __forceinline__ void stage(float* s_x, int pitch, int64_t r0, int rows) const {
    const int F = d.F, total = rows * F;
    const bool rows_fast = (d.s0 < 0 ? -d.s0 : d.s0) < (d.s1 < 0 ? -d.s1 : d.s1);
    if (rows_fast) for (int i = threadIdx.x; i < total; i += blockDim.x) { const int f = i / rows, r = i - f * rows; s_x[r * pitch + f] = load_x<T>(d, r0 + r, f); }
    else for (int i = threadIdx.x; i < total; i += blockDim.x) { const int r = i / F, f = i - r * F; s_x[r * pitch + f] = load_x<T>(d, r0 + r, f); }
  }
  __device__ __forceinline__ float at(int64_t r, int f) const { return f < d.F ? load_x<T>(d, r, f) : __int_as_float(0x7fc00000); }
};
// A CSR input: a tile's rows are NaN-filled, then each warp scatters one row at a time.  A column repeated inside a row keeps
// its last value: within 32 entries only the highest lane of each column stores, and the 32-entry steps are ordered by __syncwarp.
struct CsrSrc {
  InputDesc d;
  __device__ __forceinline__ void stage(float* s_x, int pitch, int64_t r0, int rows) const {
    const float nan = __int_as_float(0x7fc00000);
    for (int i = threadIdx.x; i < rows * pitch; i += blockDim.x) s_x[i] = nan;
    __syncthreads();
    const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    const float* vals = static_cast<const float*>(d.ptr);
    for (int r = threadIdx.x >> 5; r < rows; r += warps) {
      const int64_t a = d.indptr[r0 + r], z = d.indptr[r0 + r + 1];
      for (int64_t j0 = a; j0 < z; j0 += 32) {
        const int64_t j = j0 + lane;
        const unsigned c = j < z ? (unsigned)d.indices[j] : 0xffffffffu;
        const unsigned same = __match_any_sync(0xffffffffu, c);
        if (j < z && (same >> lane) == 1u) s_x[r * pitch + c] = vals[j];
        __syncwarp();
      }
    }
  }
  __device__ __forceinline__ float at(int64_t r, int f) const {
    const float* vals = static_cast<const float*>(d.ptr);
    for (int64_t j = d.indptr[r + 1] - 1; j >= d.indptr[r]; --j) if (d.indices[j] == f) return vals[j];
    return __int_as_float(0x7fc00000);
  }
};

}  // namespace b200
#endif
