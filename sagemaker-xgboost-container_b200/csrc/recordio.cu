// recordio.cu -- recordio-protobuf bodies (application/x-recordio-protobuf) decoded on the device into the DMatrix.
// Replaces read_recordio_protobuf + xgb.DMatrix(features, label=labels) of the container: encoder.recordio_protobuf_to_dmatrix
// (serve_utils.py:144-145 for inference requests) and data_utils.get_recordio_protobuf_dmatrix (data_utils.py:450-453 for
// training channels).  The reference parses one protobuf Record per record in Python and stacks 1-row arrays / csr_matrix rows.
//
// Wire format (DESIGN.md "recordio-protobuf"): records are [u32 magic 0xCED7230A][u32 length][payload padded to 4 bytes];
// the payload is an aialgs.data.Record (proto2): features = 1 and label = 2 are map<string, Value> (entry key = 1, value = 2),
// Value is a oneof float32_tensor = 2 / float64_tensor = 3 / int32_tensor = 7 / bytes = 9, and a tensor has packed
// values = 1, keys = 2 (uint64) and shape = 3 (uint64).  Only features["values"] and label["values"] are read.
//
// Stages: (1) the record index -- the header walk is a serial chain, done by a host thread while the body crosses PCIe;
// (2) pass 1, one warp per record: the tag walk runs on every lane (uniform control flow), packed varint arrays are walked 32
// bytes per step with a ballot over the continuation bits; it validates the record the way protobuf would, and yields the
// row kind, width, entry and label counts; (3) one exclusive scan of (rows, entries, labels); (4) pass 2, one warp per record,
// writes dense rows straight into X, or a sparse batch as CSR arrays that the scatter of DMatrix::from_csr densifies.
// Anything protobuf accepts but this fast path does not decide (unpacked or repeated fields, merged messages, a "values" key
// given twice, a malformed message ...) raises the host-route status, and the package's Python walker decides instead.
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <cub/cub.cuh>
#include "booster.h"

namespace b200 {

namespace {
constexpr unsigned kMagic = 0xCED7230Au;
constexpr unsigned kFull = 0xffffffffu;
enum TensorType { kNone = 0, kF32 = 1, kF64 = 2, kI32 = 3 };

struct Span { const unsigned char* p; unsigned len; };

struct RecInfo {                                   // pass 1 -> pass 2, one per record
  unsigned long long voff, koff, loff;             // byte offsets in the body of the packed feature values / keys / label values
  unsigned vlen, klen, llen;
  unsigned char kind, vtype, ltype, pad;           // kind: 0 skipped, 1 dense row, 2 sparse row
};
struct Cnt { long long rows, ent, lab; };          // kept rows, CSR entries (sparse batch), label values
struct CntSum { __host__ __device__ Cnt operator()(const Cnt& a, const Cnt& b) const { return Cnt{a.rows + b.rows, a.ent + b.ent, a.lab + b.lab}; } };
// widths: min / max over all kept rows, min over the rows of non-zero width; first record of non-zero width, last of width 0
struct RecGlobal { unsigned long long wmin, wmax, wmin_nz; long long first_nz, last_zero; int host, any_sparse, any_dense, unsorted; };

__device__ __forceinline__ unsigned lanemask_lt(int lane) { return (1u << lane) - 1u; }

// 4 unaligned bytes from two aligned words (the body buffer has 16 bytes of padding past its end)
__device__ __forceinline__ unsigned ld_u32(const unsigned char* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const unsigned* w = reinterpret_cast<const unsigned*>(a & ~(uintptr_t)3);
  const unsigned sh = (unsigned)(a & 3) * 8;
  return sh ? __funnelshift_r(w[0], w[1], sh) : w[0];
}

// one varint at p; returns the bytes it takes, 0 when it runs past e or over 10 bytes
__device__ int get_varint(const unsigned char* p, const unsigned char* e, unsigned long long* v) {
  unsigned long long r = 0;
  for (int i = 0; i < 10; ++i) {
    if (p + i >= e) return 0;
    const unsigned b = p[i];
    r |= (unsigned long long)(b & 0x7fu) << (7 * i);
    if (!(b & 0x80u)) { *v = r; return i + 1; }
  }
  return 0;
}

// next field of the message [p, e): 1 = a field (a length-delimited one's payload in *body), 0 = end, -1 = malformed (or a group)
__device__ int next_field(const unsigned char*& p, const unsigned char* e, unsigned* fnum, unsigned* wt, Span* body) {
  if (p >= e) return 0;
  unsigned long long tag = 0, v = 0;
  int k = get_varint(p, e, &tag);
  if (!k || tag > 0xffffffffull || (tag >> 3) == 0) return -1;
  p += k; *fnum = (unsigned)(tag >> 3); *wt = (unsigned)(tag & 7);
  switch (*wt) {
    case 0: k = get_varint(p, e, &v); if (!k) return -1; p += k; return 1;
    case 1: if (e - p < 8) return -1; p += 8; return 1;
    case 5: if (e - p < 4) return -1; p += 4; return 1;
    case 2: k = get_varint(p, e, &v); if (!k) return -1; p += k;
            if (v > (unsigned long long)(e - p)) return -1;
            body->p = p; body->len = (unsigned)v; p += v; return 1;
    default: return -1;
  }
}

// Lane-parallel walk of a packed varint array: 32 bytes per step; the bytes with the top bit clear end a varint (one ballot), and
// the lane holding such a byte decodes its varint backwards to the previous end.  fn(has, j, v) runs on every lane (has = this
// lane ends varint number j).  Returns false when a varint is longer than 10 bytes or the array ends inside one.
template <class Fn>
__device__ bool warp_varints(const unsigned char* a, unsigned len, int lane, Fn&& fn) {
  unsigned count = 0; long long last = -1; bool bad = false;
  for (unsigned base = 0; base < len; base += 32) {
    const unsigned i = base + lane;
    const unsigned b = i < len ? a[i] : 0x80u;
    const unsigned term = __ballot_sync(kFull, !(b & 0x80u));
    const bool has = (term >> lane) & 1u;
    unsigned long long v = 0;
    if (has) {
      const unsigned lower = term & lanemask_lt(lane);
      const long long start = lower ? (long long)base + (31 - __clz(lower)) + 1 : last + 1;
      if ((long long)i - start >= 10) bad = true;
      else for (long long k = i; k >= start; --k) v = (v << 7) | (a[k] & 0x7fu);
    }
    fn(has, count + __popc(term & lanemask_lt(lane)), v);
    count += __popc(term);
    if (term) last = (long long)base + (31 - __clz(term));
  }
  if (len && last != (long long)len - 1) bad = true;
  return !__any_sync(kFull, bad);
}

// float32 of a wire float32 / float64 with the NaN payloads the host route produces (protobuf hands float32 values to Python as
// doubles, numpy narrows float64 to float32): a NaN comes out quiet with the top bits of its payload
__device__ __forceinline__ float f32_of_wire(unsigned u) {
  if ((u & 0x7f800000u) == 0x7f800000u && (u & 0x007fffffu)) u |= 0x00400000u;
  return __uint_as_float(u);
}
__device__ __forceinline__ float f32_of_wire64(unsigned lo, unsigned hi) {
  if ((hi & 0x7ff00000u) == 0x7ff00000u && ((hi & 0x000fffffu) | lo))
    return __uint_as_float((hi & 0x80000000u) | 0x7fc00000u | ((hi & 0x000fffffu) << 3) | (lo >> 29));
  return __double2float_rn(__hiloint2double((int)hi, (int)lo));
}

// the values of a tensor, 32 per step: fn(has, j, value as float32, value != 0 in its own type) on every lane
template <class Fn>
__device__ bool warp_values(int type, const unsigned char* a, unsigned len, int lane, Fn&& fn) {
  if (type == kI32)
    return warp_varints(a, len, lane, [&](bool has, unsigned j, unsigned long long v) { const int x = (int)(unsigned)v; fn(has, j, __int2float_rn(x), x != 0); });
  const unsigned sz = type == kF64 ? 8u : 4u;
  if (len % sz) return false;
  const unsigned n = len / sz;
  for (unsigned base = 0; base < n; base += 32) {
    const unsigned j = base + lane;
    const bool has = j < n;
    float f = 0.0f; bool nz = false;
    if (has) {
      if (sz == 4) { const unsigned u = ld_u32(a + 4ull * j); f = f32_of_wire(u); nz = (u & 0x7fffffffu) != 0; }
      else { const unsigned lo = ld_u32(a + 8ull * j), hi = ld_u32(a + 8ull * j + 4); f = f32_of_wire64(lo, hi); nz = ((hi & 0x7fffffffu) | lo) != 0; }
    }
    fn(has, j, f, nz);
  }
  return true;
}

struct ValueInfo {
  bool ok; int type;                               // type kNone: no tensor (bytes, or nothing set)
  Span vals, keys;
  unsigned nvals, nnz, nkeys;
  unsigned long long maxkey, shape0; bool has_shape, increasing;
};

// a Value message, validated as protobuf parses it; its tensor's arrays are counted lane-parallel
__device__ ValueInfo walk_value(Span v, int lane) {
  ValueInfo r{}; r.ok = true; r.increasing = true;
  const unsigned char* p = v.p; const unsigned char* e = v.p + v.len;
  unsigned f, wt; Span b{}, t{}; int set = 0, st;
  while ((st = next_field(p, e, &f, &wt, &b)) == 1) {
    if (f == 2 || f == 3 || f == 7 || f == 9) {
      if (wt != 2) { r.ok = false; break; }                       // a oneof member with another wire type: host route
      ++set; r.type = f == 2 ? kF32 : (f == 3 ? kF64 : (f == 7 ? kI32 : kNone)); t = b;
    }
  }
  if (st < 0 || set > 1) r.ok = false;                            // malformed, or oneof members given twice (protobuf merges)
  if (!r.ok || r.type == kNone) { r.type = kNone; return r; }
  Span shape{t.p, 0}; r.vals = Span{t.p, 0}; r.keys = Span{t.p, 0};
  int nv = 0, nk = 0, ns = 0;
  p = t.p; e = t.p + t.len;
  while ((st = next_field(p, e, &f, &wt, &b)) == 1) {
    if (f >= 1 && f <= 3) {
      if (wt != 2) { r.ok = false; break; }                       // unpacked encoding
      if (f == 1) { ++nv; r.vals = b; } else if (f == 2) { ++nk; r.keys = b; } else { ++ns; shape = b; }
    }
  }
  if (st < 0 || nv > 1 || nk > 1 || ns > 1) r.ok = false;         // repeated packed fields concatenate: host route
  if (!r.ok) return r;
  unsigned nvals = 0, nnz = 0;
  r.ok &= warp_values(r.type, r.vals.p, r.vals.len, lane, [&](bool has, unsigned, float, bool nz) { nvals += has; nnz += has && nz; });
  r.nvals = __reduce_add_sync(kFull, nvals); r.nnz = __reduce_add_sync(kFull, nnz);
  unsigned long long kmax = 0, prev = 0; bool have_prev = false, inc = true; unsigned nkeys = 0;
  r.ok &= warp_varints(r.keys.p, r.keys.len, lane, [&](bool has, unsigned, unsigned long long k) {
    const unsigned m = __ballot_sync(kFull, has), lower = m & lanemask_lt(lane);
    const unsigned long long pk = __shfl_sync(kFull, k, lower ? 31 - __clz(lower) : lane);
    if (has) { ++nkeys; kmax = max(kmax, k); if (lower ? k <= pk : (have_prev && k <= prev)) inc = false; }
    if (m) { prev = __shfl_sync(kFull, k, 31 - __clz(m)); have_prev = true; }
  });
  r.nkeys = __reduce_add_sync(kFull, nkeys);
  for (int o = 16; o; o >>= 1) kmax = max(kmax, __shfl_xor_sync(kFull, kmax, o));
  r.maxkey = kmax; r.increasing = !__any_sync(kFull, !inc);
  unsigned long long s0 = 0; unsigned ndim = 0;
  r.ok &= warp_varints(shape.p, shape.len, lane, [&](bool has, unsigned j, unsigned long long d) { if (has) { ++ndim; if (j == 0) s0 = d; } });
  r.has_shape = __reduce_add_sync(kFull, ndim) > 0;
  for (int o = 16; o; o >>= 1) s0 |= __shfl_xor_sync(kFull, s0, o);      // only the lane of shape[0] holds a value
  r.shape0 = s0;
  return r;
}

// a features / label map entry: is its key "values", and its Value (absent = default Value, which holds no tensor)
__device__ bool walk_map_entry(Span m, bool* is_values, Span* val, bool* has_val) {
  const unsigned char* p = m.p; const unsigned char* e = m.p + m.len;
  unsigned f, wt; Span b{}, key{m.p, 0}; int nk = 0, nv = 0, st;
  while ((st = next_field(p, e, &f, &wt, &b)) == 1) {
    if (f == 1 || f == 2) {
      if (wt != 2) return false;
      if (f == 1) { ++nk; key = b; } else { ++nv; *val = b; }
    }
  }
  if (st < 0 || nk > 1 || nv > 1) return false;
  *is_values = key.len == 6 && key.p[0] == 'v' && key.p[1] == 'a' && key.p[2] == 'l' && key.p[3] == 'u' && key.p[4] == 'e' && key.p[5] == 's';
  *has_val = nv == 1;
  return true;
}

__global__ void __launch_bounds__(256) recordio_pass1_kernel(const unsigned char* __restrict__ body, const unsigned long long* __restrict__ offs, int64_t n,
                                                             RecInfo* __restrict__ recs, Cnt* __restrict__ cnt, RecGlobal* g) {
  __shared__ RecGlobal sg;
  if (threadIdx.x == 0) sg = RecGlobal{ULLONG_MAX, 0ull, ULLONG_MAX, LLONG_MAX, -1, 0, 0, 0, 0};
  __syncthreads();
  const int lane = threadIdx.x & 31;
  RecGlobal w{ULLONG_MAX, 0ull, ULLONG_MAX, LLONG_MAX, -1, 0, 0, 0, 0};   // this warp's share (identical on every lane)
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const unsigned char* p = body + offs[r];
    const unsigned char* e = p + *reinterpret_cast<const unsigned*>(p - 4);
    bool ok = true; int nfeat = 0, nlab = 0; bool feat_has = false, lab_has = false;
    ValueInfo fv{}, lv{};
    unsigned f, wt; Span b{}; int st;
    while ((st = next_field(p, e, &f, &wt, &b)) == 1) {
      if (f != 1 && f != 2) continue;                                 // uid / metadata / configuration and unknown fields
      if (wt != 2) { ok = false; break; }
      bool is_values = false, has_val = false; Span val{b.p, 0};
      if (!walk_map_entry(b, &is_values, &val, &has_val)) { ok = false; break; }
      // every Value of both maps is parsed by protobuf, so every one is validated; the "values" ones are kept
      ValueInfo vi = has_val ? walk_value(val, lane) : ValueInfo{true, kNone};
      if (!vi.ok) { ok = false; break; }
      if (is_values) { if (f == 1) { ++nfeat; feat_has = true; fv = vi; } else { ++nlab; lab_has = true; lv = vi; } }
    }
    if (st < 0 || nfeat > 1 || nlab > 1) ok = false;                // a "values" key given twice: the map keeps the last
    RecInfo ri{}; Cnt c{0, 0, 0};
    if (ok && feat_has && fv.type != kNone) {
      unsigned long long width;
      if (fv.nkeys > 0) {
        ri.kind = 2;
        width = fv.has_shape ? fv.shape0 : fv.maxkey + 1;
        if (fv.nvals != fv.nkeys || fv.maxkey >= width || width > (unsigned long long)INT_MAX) ok = false;   // the host route decides
        w.any_sparse = 1;
        if (!fv.increasing) w.unsorted = 1;
        c.ent = fv.nkeys;
      } else {
        ri.kind = 1; width = fv.nvals; w.any_dense = 1; c.ent = fv.nnz;
      }
      w.wmin = min(w.wmin, width); w.wmax = max(w.wmax, width);
      if (width) { w.wmin_nz = min(w.wmin_nz, width); w.first_nz = min(w.first_nz, (long long)r); } else w.last_zero = max(w.last_zero, (long long)r);
      c.rows = 1;
      ri.vtype = (unsigned char)fv.type; ri.voff = (unsigned long long)(fv.vals.p - body); ri.vlen = fv.vals.len;
      ri.koff = (unsigned long long)(fv.keys.p - body); ri.klen = fv.keys.len;
      if (lab_has && lv.type != kNone) { ri.ltype = (unsigned char)lv.type; ri.loff = (unsigned long long)(lv.vals.p - body); ri.llen = lv.vals.len; c.lab = lv.nvals; }
    }
    if (!ok) { w.host = 1; ri.kind = 0; c = Cnt{0, 0, 0}; }
    if (lane == 0) { recs[r] = ri; cnt[r] = c; }
  }
  if (lane == 0) {
    atomicMin(&sg.wmin, w.wmin); atomicMax(&sg.wmax, w.wmax); atomicMin(&sg.wmin_nz, w.wmin_nz);
    atomicMin(&sg.first_nz, w.first_nz); atomicMax(&sg.last_zero, w.last_zero);
    atomicOr(&sg.host, w.host); atomicOr(&sg.any_sparse, w.any_sparse); atomicOr(&sg.any_dense, w.any_dense); atomicOr(&sg.unsorted, w.unsorted);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (sg.wmin != ULLONG_MAX) { atomicMin(&g->wmin, sg.wmin); atomicMax(&g->wmax, sg.wmax); }
    if (sg.wmin_nz != ULLONG_MAX) { atomicMin(&g->wmin_nz, sg.wmin_nz); atomicMin(&g->first_nz, sg.first_nz); }
    if (sg.last_zero >= 0) atomicMax(&g->last_zero, sg.last_zero);
    if (sg.host) atomicOr(&g->host, 1);
    if (sg.any_sparse) atomicOr(&g->any_sparse, 1);
    if (sg.any_dense) atomicOr(&g->any_dense, 1);
    if (sg.unsorted) atomicOr(&g->unsorted, 1);
  }
}

// dense batch: row -> X[row][0, F); sparse batch: row -> CSR entries (a dense row keeps its non-zero values, as scipy's stacking
// of a dense block does); labels -> lab[]
__global__ void __launch_bounds__(256) recordio_pass2_kernel(const unsigned char* __restrict__ body, const RecInfo* __restrict__ recs, const Cnt* __restrict__ at,
                                                             int64_t n, int sparse, int F, float* __restrict__ X, unsigned long long* __restrict__ ptr,
                                                             unsigned* __restrict__ idx, float* __restrict__ val, float* __restrict__ lab) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const RecInfo ri = recs[r];
    if (ri.kind == 0) continue;
    const Cnt c = at[r];
    if (ri.llen) warp_values(ri.ltype, body + ri.loff, ri.llen, lane, [&](bool has, unsigned j, float v, bool) { if (has) lab[c.lab + j] = v; });
    const unsigned char* vp = body + ri.voff;
    if (!sparse) {
      float* row = X + c.rows * (int64_t)F;
      warp_values(ri.vtype, vp, ri.vlen, lane, [&](bool has, unsigned j, float v, bool) { if (has) row[j] = v; });
      continue;
    }
    if (lane == 0) ptr[c.rows] = (unsigned long long)c.ent;
    if (ri.kind == 2) {
      warp_varints(body + ri.koff, ri.klen, lane, [&](bool has, unsigned j, unsigned long long k) { if (has) idx[c.ent + j] = (unsigned)k; });
      warp_values(ri.vtype, vp, ri.vlen, lane, [&](bool has, unsigned j, float v, bool) { if (has) val[c.ent + j] = v; });
    } else {
      long long o = c.ent;
      warp_values(ri.vtype, vp, ri.vlen, lane, [&](bool has, unsigned j, float v, bool nz) {
        const unsigned m = __ballot_sync(kFull, has && nz);
        if (has && nz) { const long long k = o + __popc(m & lanemask_lt(lane)); idx[k] = j; val[k] = v; }
        o += __popc(m);
      });
    }
  }
}

// body-sized scratch kept across calls (a serving process decodes one request after another): no cudaMalloc per request
struct RecordioScratch {
  DevBuf<unsigned char> body, tmp; DevBuf<unsigned long long> offs, ptr; DevBuf<RecInfo> recs; DevBuf<Cnt> cnt, at;
  DevBuf<RecGlobal> g; DevBuf<unsigned> idx; DevBuf<float> val; std::vector<unsigned long long> h_offs;
};
RecordioScratch& recordio_scratch() { static thread_local RecordioScratch s; return s; }

// the record index: payload offsets of the records in order; *bad = 1 bad magic / 2 record past the end, at header offset *bad_at
void index_records(const unsigned char* b, int64_t len, std::vector<unsigned long long>* offs, int* bad, int64_t* bad_at) {
  int64_t off = 0;
  while (off + 8 <= len) {                                          // 1 to 7 trailing bytes are ignored
    unsigned magic, length;
    memcpy(&magic, b + off, 4); memcpy(&length, b + off + 4, 4);
    if (magic != kMagic) { *bad = 1; *bad_at = off; return; }
    off += 8;
    const int64_t padded = ((int64_t)length + 3) / 4 * 4;
    if (off + padded > len) { *bad = 2; *bad_at = off; return; }
    offs->push_back((unsigned long long)off);
    off += padded;
  }
}
}  // namespace

std::unique_ptr<DMatrix> DMatrix::from_recordio(const char* buf, int64_t len, int* status, std::string* message) {
  RecordioScratch& sc = recordio_scratch();
  cudaStream_t s = engine_stream();
  static const bool prof = getenv("B200XGB_RECORDIO_PROFILE") != nullptr;     // stage times on stderr (microbench/recordio_stages.py)
  auto t_last = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!prof) return;
    cudaStreamSynchronize(s);
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[recordio] %-26s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t_last).count());
    t_last = now;
  };
  *status = 0; message->clear();
  // (1) index on a host thread while the body crosses PCIe
  sc.body.ensure((size_t)len + 16);
  sc.h_offs.clear();
  int bad = 0; int64_t bad_at = 0; double walk_ms = 0.0;
  std::thread walker([&] {
    auto t0 = std::chrono::steady_clock::now();
    index_records(reinterpret_cast<const unsigned char*>(buf), len, &sc.h_offs, &bad, &bad_at);
    walk_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  });
  const cudaError_t copy = len ? cudaMemcpyAsync(sc.body.p, buf, (size_t)len, cudaMemcpyHostToDevice, s) : cudaSuccess;
  walker.join();
  CUDA_OK(copy);
  if (prof) fprintf(stderr, "[recordio] %-26s %8.3f ms\n", "index walk (host thread)", walk_ms);
  lap("h2d of the body + index");
  const int64_t n = (int64_t)sc.h_offs.size();
  B200_CHECK(n < (int64_t)0x7fffffff, "DMatrix: more than 2^31-1 rows per GPU are not supported");
  // (2) pass 1 and (3) the scan
  sc.offs.ensure((size_t)n + 1); sc.recs.ensure((size_t)n + 1); sc.cnt.ensure((size_t)n + 1); sc.at.ensure((size_t)n + 1); sc.g.ensure(1);
  if (n) CUDA_OK(cudaMemcpyAsync(sc.offs.p, sc.h_offs.data(), sizeof(unsigned long long) * n, cudaMemcpyHostToDevice, s));
  const RecGlobal g0{ULLONG_MAX, 0ull, ULLONG_MAX, LLONG_MAX, -1, 0, 0, 0, 0};
  CUDA_OK(cudaMemcpyAsync(sc.g.p, &g0, sizeof g0, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemsetAsync(sc.cnt.p + n, 0, sizeof(Cnt), s));
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)engine_num_sms() * 32));
  if (n) { recordio_pass1_kernel<<<grid, 256, 0, s>>>(sc.body.p, sc.offs.p, n, sc.recs.p, sc.cnt.p, sc.g.p); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
  size_t tmp_bytes = 0;
  CUDA_OK(cub::DeviceScan::ExclusiveScan(nullptr, tmp_bytes, sc.cnt.p, sc.at.p, CntSum(), Cnt{0, 0, 0}, (int)(n + 1), s));
  sc.tmp.ensure(tmp_bytes);
  CUDA_OK(cub::DeviceScan::ExclusiveScan(sc.tmp.p, tmp_bytes, sc.cnt.p, sc.at.p, CntSum(), Cnt{0, 0, 0}, (int)(n + 1), s)); ++g_kernel_launches;
  RecGlobal g{}; Cnt tot{};
  CUDA_OK(cudaMemcpyAsync(&g, sc.g.p, sizeof g, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(&tot, sc.at.p + n, sizeof tot, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("pass 1 + scan");
  // the decisions, in the order the reference meets them: records in order (a record protobuf or scipy would treat specially
  // comes before a framing error further on), then the stacking
  if (g.host) { *status = 2; return nullptr; }
  if (bad) { *status = 1; *message = (bad == 1 ? "Invalid RecordIO magic at offset " : "Truncated record at offset ") + std::to_string(bad_at); return nullptr; }
  if (tot.rows == 0) { *status = 1; *message = "No records found in RecordIO-Protobuf data"; return nullptr; }
  const bool sparse = g.any_sparse != 0;
  // np.vstack wants equal lengths; scipy's block stacking takes the column width from the first block that has one, so in a
  // sparse batch rows of width 0 are accepted ahead of the first row of width W, every other row must have width W
  if (sparse ? (g.wmin_nz != g.wmax || g.last_zero > g.first_nz) : g.wmin != g.wmax) {
    *status = 1;
    *message = sparse ? "recordio-protobuf: rows of a sparse batch have different widths (" + std::to_string(g.wmin) + " and " + std::to_string(g.wmax) +
                        "; a tensor without keys is a dense row of len(values) entries, width 0 only ahead of the first wider row): scipy.sparse.vstack raises"
                      : "recordio-protobuf: dense rows have different lengths (" + std::to_string(g.wmin) + " and " + std::to_string(g.wmax) + "): np.vstack raises";
    return nullptr;
  }
  if (sparse && g.any_dense && g.unsorted) { *status = 2; return nullptr; }   // scipy sums repeated keys when dense rows join the batch
  const int64_t rows = tot.rows;
  const int F = (int)g.wmax;
  // (4) pass 2
  auto dm = std::make_unique<DMatrix>();
  dm->n = rows; dm->F = F;
  dm->X.alloc((size_t)rows * F);
  dm->d_labels.alloc((size_t)tot.lab);
  unsigned long long ent_total = (unsigned long long)tot.ent;
  if (sparse) {
    sc.ptr.ensure((size_t)rows + 1); sc.idx.ensure((size_t)std::max<long long>(tot.ent, 1)); sc.val.ensure((size_t)std::max<long long>(tot.ent, 1));
    CUDA_OK(cudaMemcpyAsync(sc.ptr.p + rows, &ent_total, sizeof ent_total, cudaMemcpyHostToDevice, s));
  }
  recordio_pass2_kernel<<<grid, 256, 0, s>>>(sc.body.p, sc.recs.p, sc.at.p, n, sparse ? 1 : 0, F, dm->X.p, sc.ptr.p, sc.idx.p, sc.val.p, dm->d_labels.p);
  ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  lap("pass 2");
  if (sparse) csr_to_dense_device(sc.ptr.p, sc.idx.p, sc.val.p, rows, F, dm->X.p, s);
  lap("scatter");
  dm->labels.resize((size_t)tot.lab);
  if (tot.lab) CUDA_OK(cudaMemcpyAsync(dm->labels.data(), dm->d_labels.p, sizeof(float) * tot.lab, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  dm->finish_upload(std::nanf(""));
  lap("labels + missing count");
  return dm;
}

}  // namespace b200
