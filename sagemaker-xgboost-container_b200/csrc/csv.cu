// csv.cu -- device-side CSV -> float32 matrix for the serving path (SURVEY.md section 8f row 1).
// Replaces the Python split + np.array(...).astype(float) of the container's encoder.csv_to_dmatrix (encoder.py:31-52),
// reached from algorithm_mode/serve_utils.py:121-131 (parse_content_data) for every text/csv invocation request.
//
// Semantics kept from that code path: rows are separated by '\n' (payload already stripped of leading/trailing
// whitespace), fields by one delimiter character, an empty field is NaN, every row must have the same number of
// fields, a field is what Python's float() accepts (decimal, exponent, inf/nan in any case).  Values take the same two
// roundings: text -> nearest double (Clinger's exact fast path: <= 19 significant digits below 2^53 and |exp10| <= 22,
// one IEEE multiply or divide) -> nearest float32 (what xgb.DMatrix does with a float64 array).  A field outside the fast
// path (or malformed) raises a flag and the caller falls back to the host parser, so results never differ.  The byte-level
// code (field literals, newline count, libsvm token walk) is in text_parse.h, shared with a CPU sweep of the tests.
//
// Kernels: (1) newline count, (2) newline positions (CUB select), (3) one thread per row walks its fields.  Text is read
// once from HBM (L1-cached byte loads; rows are short and contiguous per thread).  The row table of (2) has as many entries
// as (1) counted only if the two agree: the parse kernels compare the select's own count with it before they read a row
// bound, and on a mismatch write kRowTableMismatch and return.  The host raises on that code (a device bug, not a body the
// host route should see), without an extra synchronisation.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cub/cub.cuh>
#include <cstring>
#include "booster.h"
#include "text_parse.h"

namespace b200 {

struct IsNewline {
  const char* text;
  __host__ __device__ bool operator()(const int64_t& i) const { return text[i] == '\n'; }
};

// err code of a row table whose select count differs from the newline count (never a property of the body)
constexpr int kRowTableMismatch = 16;

// one thread per row: row r covers [start, end) where start = r ? nl[r-1] + 1 : 0 and end = r < n-1 ? nl[r] : len;
// num_nl is the select's count of the entries it wrote into nl
__global__ void __launch_bounds__(256) csv_parse_kernel(const char* text, int64_t len, const int64_t* nl, const long long* num_nl, int64_t n, int F,
                                                        char delim, float* out, int* err) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (*num_nl != n - 1) { if (r == 0) atomicMax(err, kRowTableMismatch); return; }
  const char* p = text + (r ? nl[r - 1] + 1 : 0);
  const char* e = text + (r < n - 1 ? nl[r] : len);
  float* o = out + r * F;
  int f = 0;
  const char* tok = p;
  for (const char* q = p;; ++q) {
    if (q >= e || *q == delim) {
      if (f < F) { float v; if (!parse_field(tok, q, &v)) { atomicMax(err, 2); v = 0.f; } o[f] = v; }
      ++f; tok = q + 1;
      if (q >= e) break;
    }
  }
  if (f != F) atomicMax(err, 1);                                                   // ragged row
}

// newline count: 16 B per thread per step
__global__ void __launch_bounds__(256) count_newlines_kernel(const char* text, int64_t len, unsigned long long* out) {
  unsigned long long c = 0;
  const int64_t nvec = len / 16;
  const uint4* v = reinterpret_cast<const uint4*>(text);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const uint4 w = v[i];
    const unsigned ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c += newlines_in_word(ws[k]);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) for (int64_t i = nvec * 16; i < len; ++i) c += text[i] == '\n';
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

__global__ void fill_value_kernel(float* X, int64_t count, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) X[i] = v;
}

// request-sized scratch kept across calls (a serving process parses one body after another): no cudaMalloc per request
struct CsvScratch { DevBuf<char> text; DevBuf<int64_t> nl; DevBuf<unsigned char> tmp; DevBuf<unsigned long long> cnt; DevBuf<int> err; };
static CsvScratch& csv_scratch() { static thread_local CsvScratch s; return s; }

// the select's count of newline positions, in device memory (zero when no select ran: nnl == 0)
static const long long* newline_select_count(CsvScratch& sc) { return reinterpret_cast<const long long*>(sc.cnt.p + 1); }

// newline count, then (for nnl > 0) their positions into sc.nl; the count is on the host when this returns.  lap(stage)
// after each of the two steps (profiling).
template <class Lap>
static unsigned long long newline_table(CsvScratch& sc, int64_t len, cudaStream_t s, Lap&& lap) {
  CUDA_OK(cudaMemsetAsync(sc.cnt.p, 0, 16, s));
  count_newlines_kernel<<<engine_num_sms() * 8, 256, 0, s>>>(sc.text.p, len, sc.cnt.p); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  unsigned long long nnl = 0;
  CUDA_OK(cudaMemcpyAsync(&nnl, sc.cnt.p, sizeof(nnl), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("count newlines");
  sc.nl.ensure((size_t)nnl + 1);
  if (nnl > 0) {                                                                   // positions of the newlines, in order
    cub::CountingInputIterator<int64_t> idx(0);
    IsNewline pred{sc.text.p};
    size_t tmp_bytes = 0;
    long long* d_num = reinterpret_cast<long long*>(sc.cnt.p + 1);
    CUDA_OK(cub::DeviceSelect::If(nullptr, tmp_bytes, idx, sc.nl.p, d_num, len, pred, s));
    sc.tmp.ensure(tmp_bytes);
    CUDA_OK(cub::DeviceSelect::If(sc.tmp.p, tmp_bytes, idx, sc.nl.p, d_num, len, pred, s));
    ++g_kernel_launches;
  }
  lap("newline positions");
  return nnl;
}

// a parse kernel found the row table inconsistent with the newline count: a device bug, so no host-route fallback
[[noreturn]] static void raise_row_table_mismatch(CsvScratch& sc, unsigned long long nnl, cudaStream_t s) {
  long long selected = 0;
  CUDA_OK(cudaMemcpyAsync(&selected, newline_select_count(sc), sizeof selected, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  throw Error("text parser: the newline count (" + std::to_string(nnl) + ") differs from the newline positions found (" +
              std::to_string(selected) + ")");
}

// returns 0 = ok, 1 = ragged rows, 2 = a field outside the exact fast path / malformed (caller falls back to the host parser)
int parse_csv_device(const char* h_text, int64_t len, char delim, int F, int64_t* n_rows_out, DevBuf<float>* X, cudaStream_t s) {
  CsvScratch& sc = csv_scratch();
  static const bool prof = getenv("B200XGB_CSV_PROFILE") != nullptr;          // stage times on stderr (microbench/csv_stages.py)
  auto t_last = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!prof) return;
    cudaStreamSynchronize(s);
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[csv] %-22s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t_last).count());
    t_last = now;
  };
  sc.text.ensure((size_t)len + 16); sc.cnt.ensure(2); sc.err.ensure(1);
  CUDA_OK(cudaMemcpyAsync(sc.text.p, h_text, (size_t)len, cudaMemcpyHostToDevice, s));
  lap("h2d of the text");
  CUDA_OK(cudaMemsetAsync(sc.err.p, 0, 4, s));
  const unsigned long long nnl = newline_table(sc, len, s, lap);
  const int64_t n = (int64_t)nnl + 1;
  *n_rows_out = n;
  X->alloc((size_t)n * F);
  lap("alloc X");
  csv_parse_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(sc.text.p, len, sc.nl.p, newline_select_count(sc), n, F, delim, X->p, sc.err.p);
  ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  int err = 0;
  CUDA_OK(cudaMemcpyAsync(&err, sc.err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("parse kernel");
  if (err == kRowTableMismatch) raise_row_table_mismatch(sc, nnl, s);
  return err;
}

// ---------------------------------------------------------------------------------------------------------------------
// libsvm request bodies ("label idx:val idx:val ..." per line): serve_utils._get_sparse_matrix_from_libsvm
// (algorithm_mode/serve_utils.py:94-118, per-token Python loop -> COO -> csr_matrix -> DMatrix: absent entries are MISSING) and
// encoder.libsvm_to_dmatrix (encoder.py:54-86, script mode: dense zeros, absent entries are 0.0).  Both shift the indices to
// 0-based when the smallest index in the body is >= 1.  One thread per line, two passes over the text: (1) index range and
// entry check, (2) values into the pre-filled matrix.  Anything the two Python routes treat specially -- an index that is not
// plain digits, a value outside the exact fast path or empty, an index repeated inside a line (COO sums it, the dict keeps the
// last), a token with a second ':' -- raises the fallback flag and the caller takes the reference's own host route.
struct LibsvmRange { int min_idx, max_idx; unsigned long long entries; int err; int last_row_entries; };

template <bool kFill>
__global__ void __launch_bounds__(256) libsvm_kernel(const char* text, int64_t len, const int64_t* nl, const long long* num_nl, int64_t n, LibsvmRange* rg,
                                                     int whitespace_mode, float* X, int F, int shift, float absent) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (*num_nl != n - 1) { if (r == 0) atomicMax(&rg->err, kRowTableMismatch); return; }
  const char* p = text + (r ? nl[r - 1] + 1 : 0);
  const char* e = text + (r < n - 1 ? nl[r] : len);
  int lo = 0x7fffffff, hi = -1, cnt = 0;
  const bool good = libsvm_line(p, e, whitespace_mode, [&](int idx, float val) {
    ++cnt; lo = min(lo, idx); hi = max(hi, idx);
    if (!kFill) return true;
    float* slot = X + r * F + (idx - shift);
    // serve_utils' COO -> CSR conversion SUMS an index repeated inside a line (the encoder's dict keeps the last one, which is
    // what this sequential walk does): with NaN as the fill value a slot that is no longer NaN has been written before
    const bool fresh = whitespace_mode || (val == val && *slot != *slot);
    *slot = val;
    return fresh;
  });
  if (!good) atomicMax(&rg->err, 2);
  if (!kFill) {
    if (cnt) { atomicMin(&rg->min_idx, lo); atomicMax(&rg->max_idx, hi); atomicAdd(&rg->entries, (unsigned long long)cnt); }
    if (r == n - 1) rg->last_row_entries = cnt;
  }
}

// status: 0 ok, 2 host route needed (see above), 3 no entries at all (both routes special-case it on the host)
int parse_libsvm_device(const char* h_text, int64_t len, int whitespace_mode, float absent, int64_t* n_rows_out, int* F_out, DevBuf<float>* X, cudaStream_t s) {
  CsvScratch& sc = csv_scratch();
  sc.text.ensure((size_t)len + 16); sc.cnt.ensure(2); sc.err.ensure(16);
  CUDA_OK(cudaMemcpyAsync(sc.text.p, h_text, (size_t)len, cudaMemcpyHostToDevice, s));
  const unsigned long long nnl = newline_table(sc, len, s, [](const char*) {});
  const int64_t n = (int64_t)nnl + 1;
  static_assert(sizeof(LibsvmRange) <= 16 * sizeof(int), "range block lives in the err scratch");
  LibsvmRange* rg = reinterpret_cast<LibsvmRange*>(sc.err.p);
  LibsvmRange init{0x7fffffff, -1, 0ull, 0, 0};
  CUDA_OK(cudaMemcpyAsync(rg, &init, sizeof init, cudaMemcpyHostToDevice, s));
  const unsigned grid = (unsigned)((n + 255) / 256);
  libsvm_kernel<false><<<grid, 256, 0, s>>>(sc.text.p, len, sc.nl.p, newline_select_count(sc), n, rg, whitespace_mode, nullptr, 0, 0, absent); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  LibsvmRange h{};
  CUDA_OK(cudaMemcpyAsync(&h, rg, sizeof h, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  if (h.err == kRowTableMismatch) raise_row_table_mismatch(sc, nnl, s);
  if (h.err != 0) return 2;
  if (h.entries == 0) return 3;
  if (!whitespace_mode && h.last_row_entries == 0) return 2;      // csr_matrix((data, (row, col))) infers its row count: trailing empty lines vanish there
  const int shift = h.min_idx >= 1 ? 1 : 0;
  const int F = h.max_idx - shift + 1;
  B200_CHECK((double)n * (double)F < 4e9, "libsvm body: the dense matrix would exceed 4e9 entries");
  X->alloc((size_t)n * F);
  fill_value_kernel<<<engine_num_sms() * 8, 256, 0, s>>>(X->p, (int64_t)n * F, absent); ++g_kernel_launches;
  libsvm_kernel<true><<<grid, 256, 0, s>>>(sc.text.p, len, sc.nl.p, newline_select_count(sc), n, rg, whitespace_mode, X->p, F, shift, absent); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(&h, rg, sizeof h, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  if (h.err != 0) return 2;
  *n_rows_out = n; *F_out = F;
  return 0;
}

std::unique_ptr<DMatrix> DMatrix::from_libsvm_text(const char* text, int64_t len, int whitespace_mode, float absent, int* status) {
  auto dm = std::make_unique<DMatrix>();
  cudaStream_t s = engine_stream();
  int64_t n = 0; int F = 0;
  *status = parse_libsvm_device(text, len, whitespace_mode, absent, &n, &F, &dm->X, s);
  if (*status != 0) return nullptr;
  B200_CHECK(n < (int64_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  dm->n = n; dm->F = F;
  dm->finish_upload(std::nanf(""));
  return dm;
}

// training channels (data_utils.py:289-318: "?format=csv&label_column=0[&weight_column=1]"): the label / weight columns
// leave the parsed matrix on the device, the remaining columns are compacted in place order
__global__ void __launch_bounds__(256) split_columns_kernel(const float* in, int64_t n, int Fin, int label_col, int weight_col, float* out, float* y, float* w) {
  const int Fout = Fin - (label_col >= 0 ? 1 : 0) - (weight_col >= 0 ? 1 : 0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * Fin; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / Fin; const int c = (int)(i - r * Fin);
    const float v = in[i];
    if (c == label_col) y[r] = v;
    else if (c == weight_col) w[r] = v;
    else out[r * Fout + c - (label_col >= 0 && c > label_col ? 1 : 0) - (weight_col >= 0 && c > weight_col ? 1 : 0)] = v;
  }
}

std::unique_ptr<DMatrix> DMatrix::from_csv_text_labeled(const char* text, int64_t len, char delim, int label_col, int weight_col, int* status) {
  int Fin = 1;
  for (int64_t i = 0; i < len && text[i] != '\n'; ++i) if (text[i] == delim) ++Fin;
  B200_CHECK(label_col < Fin && weight_col < Fin && (label_col < 0 || label_col != weight_col), "CSV: label_column / weight_column out of range");
  cudaStream_t s = engine_stream();
  DevBuf<float> raw; int64_t n = 0;
  *status = parse_csv_device(text, len, delim, Fin, &n, &raw, s);
  if (*status != 0) return nullptr;
  B200_CHECK(n < (int64_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  auto dm = std::make_unique<DMatrix>();
  const int Fout = Fin - (label_col >= 0 ? 1 : 0) - (weight_col >= 0 ? 1 : 0);
  dm->n = n; dm->F = Fout;
  dm->X.alloc((size_t)n * std::max(Fout, 0));
  DevBuf<float> dy, dw; dy.alloc(label_col >= 0 ? n : 0); dw.alloc(weight_col >= 0 ? n : 0);
  const int grid = (int)std::min<int64_t>((n * Fin + 255) / 256, engine_num_sms() * 32);
  split_columns_kernel<<<grid, 256, 0, s>>>(raw.p, n, Fin, label_col, weight_col, dm->X.p, dy.p, dw.p); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  std::vector<float> hy(label_col >= 0 ? n : 0), hw(weight_col >= 0 ? n : 0);
  if (!hy.empty()) CUDA_OK(cudaMemcpyAsync(hy.data(), dy.p, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  if (!hw.empty()) CUDA_OK(cudaMemcpyAsync(hw.data(), dw.p, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  dm->finish_upload(std::nanf(""));
  if (!hy.empty()) dm->set_float_info("label", hy.data(), hy.size());
  if (!hw.empty()) dm->set_float_info("weight", hw.data(), hw.size());
  return dm;
}

std::unique_ptr<DMatrix> DMatrix::from_csv_text(const char* text, int64_t len, char delim, int* status) {
  // columns from the first line (the container sniffs the delimiter there too, encoder.py:46-48)
  int F = 1;
  for (int64_t i = 0; i < len && text[i] != '\n'; ++i) if (text[i] == delim) ++F;
  auto dm = std::make_unique<DMatrix>();
  cudaStream_t s = engine_stream();
  int64_t n = 0;
  *status = parse_csv_device(text, len, delim, F, &n, &dm->X, s);
  if (*status != 0) return nullptr;
  B200_CHECK(n < (int64_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  dm->n = n; dm->F = F;
  dm->finish_upload(std::nanf(""));
  return dm;
}

}  // namespace b200
