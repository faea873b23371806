// hist.cu -- per-node gradient/hessian histogram build: THE hot kernel (SURVEY.md section 8a row A7).
// Replaces upstream xgboost's BuildHist (src/common/hist_util.cc / src/tree/gpu_hist/histogram.cu),
// reached from the container at algorithm_mode/train.py:367-376 (xgb.train -> Booster.update).
//
// Design (DESIGN.md "histogram kernels"; measurements in profiles/):
//  * sm_90a has exactly one fast shared-memory atomic: 32-bit integer ATOMS.ADD (float and 64-bit adds compile to
//    ATOMS.CAST.SPIN CAS loops), and it runs at full rate only when the 32 lanes of the instruction hit 32 distinct
//    banks.  So the histogram of one 32-feature group is int32 planes [256 bins][32 slots]: bank == slot, and every
//    instruction below has its lanes on 32 distinct slots (per-row slot rotation, see LaneConst).
//  * Layout without pad work: features live in FULL 32-wide groups plus a narrow tail (F = 100 -> 3 groups + 4-wide
//    tail), so no atomic and no HBM byte is spent on pad slots (round 1: 4 groups x 25 of 32 slots = 22 % waste).
//  * Two kernels share the accumulate / spill code:
//      hist_root_kernel    the contiguous root pass.  A producer thread streams row tiles with TMA (2-D tensor map for
//                          the main block: cp.async.bulk.tensor -> UTMALDG, 1-D bulk copies for (g,h) and the tail:
//                          UBLKCP) into an mbarrier ring; consumer warps read bins with conflict-free LDS.128 and issue
//                          the atomics.  GONLY variant for constant-hessian objectives: the H plane of the root never
//                          changes between rounds, so the slot is pre-loaded with the cached H plane and only G is
//                          accumulated (1 atomic per update instead of 2); its gradients are the dense g (4 B per row).
//      hist_gather_kernel  the deeper levels: rows gathered by row id (LDG.128 per 16 B chunk straight to registers, a
//                          rolling one-super-tile-ahead prefetch), (g,h) read by POSITION (they travel with the row
//                          ids through the partition; g alone for constant-hessian objectives, whose h_q is a constant),
//                          tail bytes from the pad of the row's line-aligned copy where there is one.
//  * Gradients are rounded to a power-of-two fixed-point grid (|g_q| <= 2^18, h_q <= 2^19) so a window of 8064 rows per
//    CTA cannot overflow int32; between windows, accumulators above 2^25 (G) / 2^26 (H) are spilled to the global int64 histogram with
//    RED.ADD.64 (sparse), and everything is flushed at the end of the CTA's portion: by the root kernel with RED.ADD.64, by the
//    gather kernel with plain stores into a partial slot per (CTA, node) segment that hist_reduce_kernel sums.  Sums are exact integers =>
//    bit-reproducible for any grid size, block schedule or GPU count; the NCCL all-reduce is order-independent.
#include <cuda.h>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>
#include "engine.h"
#include "tree.h"

namespace b200 {

constexpr int kSuperRows = 32;
constexpr int kMinRowsPerCta = 4096;              // do not pay a flush for fewer rows than this
// Between windows an accumulator is spilled only when the next window could overflow it: a window adds at most
// window * 2^bits = 2^31 - 2^25 to a G accumulator (int32) and window * 2^(bits+1) = 2^32 - 2^26 to an H accumulator (uint32;
// engine.h), so whatever stays below 2^25 / 2^26 is safe.  (A constant hessian quantises to h_q = 2^19: an H accumulator
// reaches 2^24 after 32 rows of one bin, about every window, and 2^26 after 128.)
constexpr int kSpillThresholdG = 1 << 25;
constexpr unsigned kSpillThresholdH = 1u << 26;
constexpr int kPlaneBytes = kGroupEntries * 4;    // 32 KB
constexpr int kMaxSmem = 232448;                  // 227 KB opt-in limit per CTA
// root kernel: consumer warps work in teams; a ring stage (tile of kRootRows rows) is consumed by ONE team, warp w of the team
// taking row block w (16 rows) across all groups, so per-tile synchronisation is amortised over ng units per warp
constexpr int kTeamWarps = 4, kTeams = 6, kRootRows = 16 * kTeamWarps;
constexpr int kRootConsumerWarps = kTeamWarps * kTeams;
constexpr int kRootProducerWarps = 3;                       // one issuing lane each, tiles round-robin: a single thread tops out at ~3.9 TB/s
constexpr int kRootThreads = (kRootConsumerWarps + kRootProducerWarps) * 32;      // 864 threads, <= 72 registers

// compile-time loop: the body receives std::integral_constant<int, K> (template arguments depend on the index)
template <int K, int N, typename F> __device__ __forceinline__ void static_for(F&& f) {
  if constexpr (K < N) { f(std::integral_constant<int, K>{}); static_for<K + 1, N>(f); }
}

// ---------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldg_nc_v2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ unsigned ldg_nc_u32(const void* p) {
  unsigned r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ float2 ldg_nc_f2(const void* p) {
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 lds_v4(unsigned addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ uint2 lds_v2(unsigned addr) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(addr));
  return r;
}
__device__ __forceinline__ unsigned lds_u32(unsigned addr) {
  unsigned r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(addr));
  return r;
}
__device__ __forceinline__ void red_shared_s32(unsigned addr, int v) {
  asm volatile("red.shared.add.s32 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}
template <int OFF> __device__ __forceinline__ void red_shared_s32_off(unsigned addr, int v) {       // plane offsets ride in the immediate field
  asm volatile("red.shared.add.s32 [%0+%2], %1;" :: "r"(addr), "r"(v), "n"(OFF) : "memory");
}
template <int OFF> __device__ __forceinline__ void red_shared_u32_off(unsigned addr, unsigned v) {
  asm volatile("red.shared.add.u32 [%0+%2], %1;" :: "r"(addr), "r"(v), "n"(OFF) : "memory");
}
__device__ __forceinline__ void red_shared_u32(unsigned addr, unsigned v) {
  asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void red_global_s64(long long* p, long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
// mbarrier / TMA (Hopper+ async-copy machinery; SASS: SYNCS.*, UTMALDG, UBLKCP)
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst, const CUtensorMap* tm, int c0, int c1, unsigned bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               :: "r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* tm, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" :: "l"(tm), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_load_1d(unsigned dst, const void* src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// lane -> slot schedule of a (16 rows x one 32-feature group) unit.
// Two lanes share a row: lane = 2*row + half, each holds 16 of the group's 32 bin bytes.  Step j of 16 makes the lane
// update slot 16*half + rot(j): the per-row rotation (rot = row) makes the 16 rows of an instruction touch 16 different
// slots of each half -> every ATOMS instruction hits 32 distinct banks (enumerated in tests/test_hist_lane_mapping.py).
// ---------------------------------------------------------------------------------------------
// The inner loop is issue-bound, so everything lane-constant is precomputed: A[4*jw+jb] is the complete shared-memory
// address of the slot that step (jw, jb) updates (bin 0, group 0, G plane) and S[jb] the PRMT selector of its bin byte;
// a step is PRMT + LEA + one RED per plane, with the group / plane offset in the RED's immediate field.
struct LaneConst { unsigned A[16]; unsigned S[4]; int qw; };

__device__ __forceinline__ LaneConst make_lane_const_rot(int rot, int half, unsigned smem_base) {
  LaneConst lc;
  lc.qw = rot >> 2;
  const int qb = rot & 3;
#pragma unroll
  for (int jb = 0; jb < 4; ++jb) lc.S[jb] = 0x4440u | (unsigned)((jb + qb) & 3);
#pragma unroll
  for (int jw = 0; jw < 4; ++jw)
#pragma unroll
    for (int jb = 0; jb < 4; ++jb)
      lc.A[4 * jw + jb] = smem_base + 64u * (unsigned)half + 16u * (unsigned)((jw + lc.qw) & 3) + 4u * (unsigned)((jb + qb) & 3);
  // opaque to the optimiser: otherwise it rematerialises these 20 values from their formulas inside the issue-bound loop
#pragma unroll
  for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(lc.A[i]));
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(lc.S[i]));
  return lc;
}
// (16 rows x one group) unit: two lanes per row, rotation = row
__device__ __forceinline__ LaneConst make_lane_const(int lane, unsigned smem_base) { return make_lane_const_rot(lane >> 1, lane & 1, smem_base); }

// word rotation of a 16 B chunk held in registers: ww[jw] = w[(jw + qw) & 3]
__device__ __forceinline__ void rotate_words(const LaneConst& lc, const uint4& w, unsigned (&ww)[4]) {
  unsigned w0 = w.x, w1 = w.y, w2 = w.z, w3 = w.w;
  if (lc.qw & 1) { unsigned x = w0; w0 = w1; w1 = w2; w2 = w3; w3 = x; }
  if (lc.qw & 2) { unsigned x = w0; w0 = w2; w2 = x; x = w1; w1 = w3; w3 = x; }
  ww[0] = w0; ww[1] = w1; ww[2] = w2; ww[3] = w3;
}

// The gather kernel is register-bound, not issue-bound: it rotates the BYTES of the data too (one funnel shift per word) and
// uses immediate PRMT selectors, so the four selector registers of LaneConst are never live there
__device__ __forceinline__ void rotate_words_bytes(int qw, int qb8, const uint4& w, unsigned (&ww)[4]) {
  unsigned w0 = w.x, w1 = w.y, w2 = w.z, w3 = w.w;
  if (qw & 1) { unsigned x = w0; w0 = w1; w1 = w2; w2 = w3; w3 = x; }
  if (qw & 2) { unsigned x = w0; w0 = w2; w2 = x; x = w1; w1 = w3; w3 = x; }
  ww[0] = __funnelshift_r(w0, w0, qb8); ww[1] = __funnelshift_r(w1, w1, qb8); ww[2] = __funnelshift_r(w2, w2, qb8); ww[3] = __funnelshift_r(w3, w3, qb8);
}
template <int GOFF>
__device__ __forceinline__ void accumulate16_pairs_prerotated(const unsigned (&A)[16], const unsigned (&ww)[4], int gq, unsigned hq) {
#pragma unroll
  for (int jw = 0; jw < 4; ++jw) {
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      const unsigned bin = (ww[jw] >> (8 * jb)) & 0xffu;            // byte jb of the byte-rotated word == byte (jb + qb) & 3 of the original
      const unsigned addr = (bin << 7) + A[4 * jw + jb];
      red_shared_s32_off<GOFF>(addr, gq);
      red_shared_u32_off<GOFF + 32768>(addr, hq);
    }
  }
}

// 16 conflict-free atomic (pairs) of one lane's 16 bin bytes (already word-rotated) into the planes at byte offset GOFF
template <bool GONLY, int GOFF>
__device__ __forceinline__ void accumulate16(const LaneConst& lc, const unsigned (&ww)[4], int gq, unsigned hq) {
#pragma unroll
  for (int jw = 0; jw < 4; ++jw) {
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      const unsigned bin = __byte_perm(ww[jw], 0u, lc.S[jb]);
      const unsigned addr = (bin << 7) + lc.A[4 * jw + jb];
      red_shared_s32_off<GOFF>(addr, gq);
      if (!GONLY) red_shared_u32_off<GOFF + 32768>(addr, hq);
    }
  }
}

// Tail features (tw = 4 or 8 bytes per row, one row per lane).  Plane layout [bin][trep][tw]: with trep * tw == 32 the
// replica index (from the lane) makes bank == (replica, slot) -> conflict-free; with trep == 1 (no room for replicas
// next to 200 KB of main planes) bank conflicts are data dependent but the tail is only tw of F features.
struct TailConst { unsigned base_g, hplane_bytes, bin_stride, rep_off; int tw; };

template <bool GONLY>
__device__ __forceinline__ void tail_accumulate(const TailConst& tc, int lane, unsigned w0, unsigned w1, int gq, unsigned hq) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < tc.tw) {
      const unsigned slot = (unsigned)(j + lane) & (unsigned)(tc.tw - 1);
      const unsigned bin = __byte_perm(w0, w1, slot) & 0xffu;       // selector nibbles 1..3 are 0 -> mask the replicated byte 0
      const unsigned addr = tc.base_g + bin * tc.bin_stride + tc.rep_off + slot * 4u;
      red_shared_s32(addr, gq);
      if (!GONLY) red_shared_u32(addr + tc.hplane_bytes, hq);
    }
  }
}

// Same with the tail geometry known at compile time (gather kernel: everything but the lane's base address folds into immediates)
template <int TW, int TREP>
__device__ __forceinline__ void tail_accumulate_ct(unsigned base_rep, int lane, unsigned w0, unsigned w1, int gq, unsigned hq) {
  constexpr unsigned kBinStride = (unsigned)(TW * TREP) * 4u, kHPlane = 256u * kBinStride;
#pragma unroll
  for (int j = 0; j < TW; ++j) {
    const unsigned slot = (unsigned)(j + lane) & (unsigned)(TW - 1);
    const unsigned bin = __byte_perm(w0, w1, slot) & 0xffu;
    const unsigned addr = base_rep + bin * kBinStride + slot * 4u;
    red_shared_s32(addr, gq);
    red_shared_u32(addr + kHPlane, hq);
  }
}

// warp-reduce one window's worth of per-lane (g, h) sums (32-bit is enough per window) into the node's int64 totals
__device__ __forceinline__ void flush_node_sum(GH64* dst, int g, unsigned h, int lane) {
  long long G = g, H = h;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { G += __shfl_xor_sync(0xffffffffu, G, o); H += __shfl_xor_sync(0xffffffffu, H, o); }
  if (lane == 0 && (G != 0 || H != 0)) { red_global_s64(&dst->g, G); red_global_s64(&dst->h, H); }
}

// Spill / flush pass over the CTA's accumulators.  Between windows only accumulators that could overflow in the next
// window leave for the global int64 histogram (sparse RED.ADD.64); `last` flushes everything that is non-zero.
template <int PL>      // planes per group in shared memory: 1 = G only, 2 = G then H
__device__ __forceinline__ void spill_main(int* smem, int ng_here, GH64* out, bool last, int tid, int nthr) {
  const int vecs = ng_here * PL * (kGroupEntries / 4);
  // every CTA flushes the same histogram: each one starts at a different place so that the REDs of a wave of CTAs spread over
  // the L2 slices instead of queueing on the same lines
  const int start = (int)(((long long)blockIdx.x * vecs) / gridDim.x);
  for (int i = tid; i < vecs; i += nthr) {
    int v = i + start; if (v >= vecs) v -= vecs;
    int4 x = reinterpret_cast<int4*>(smem)[v];
    if ((x.x | x.y | x.z | x.w) == 0) continue;
    const int plane = v >> 11;                                // 2048 int4 per plane
    const int e0 = (v & 2047) << 2;
    const bool is_h = PL == 2 && (plane & 1);
    GH64* o = out + (size_t)(plane / PL) * kGroupEntries + e0;
    int vals[4] = {x.x, x.y, x.z, x.w};
    bool any = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int val = vals[k];
      const bool sp = last ? (val != 0) : (is_h ? ((unsigned)val >= kSpillThresholdH) : (val >= kSpillThresholdG || val <= -kSpillThresholdG));
      if (sp) {
        red_global_s64(is_h ? &o[k].h : &o[k].g, is_h ? (long long)(unsigned)val : (long long)val);
        vals[k] = 0; any = true;
      }
    }
    if (any) reinterpret_cast<int4*>(smem)[v] = make_int4(vals[0], vals[1], vals[2], vals[3]);
  }
}

template <int PL>
__device__ __forceinline__ void spill_tail(int* tsm, int tw, int trep, GH64* out_tail, bool last, int tid, int nthr) {
  const int per_plane = 256 * tw * trep;
  const int per_bin = tw * trep;
  for (int idx = tid; idx < PL * per_plane; idx += nthr) {
    const int val = tsm[idx];
    if (val == 0) continue;
    const bool is_h = idx >= per_plane;
    const int e = is_h ? idx - per_plane : idx;
    const int bin = e / per_bin, slot = e & (tw - 1);
    const bool sp = last ? true : (is_h ? ((unsigned)val >= kSpillThresholdH) : (val >= kSpillThresholdG || val <= -kSpillThresholdG));
    if (sp) {
      GH64* o = out_tail + bin * tw + slot;
      red_global_s64(is_h ? &o->h : &o->g, is_h ? (long long)(unsigned)val : (long long)val);
      tsm[idx] = 0;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Root pass: contiguous rows, TMA-staged.  One CTA per SM; the last warp is the producer.
// ---------------------------------------------------------------------------------------------
struct RootCfg {
  int S;                   // ring stages (tiles of kRootRows rows)
  int trep;                // tail replicas in shared memory
  int box_groups;          // TMA box width / 32
  unsigned tail_off;       // byte offsets inside dynamic shared memory
  unsigned ring_off;       // (128 B aligned at run time, slack reserved)
  unsigned stage_bytes;
  unsigned total;
  int flags;               // experiment knobs (B200XGB_ROOT_FLAGS): 1 = main block by 1-D bulk copy when the tile is contiguous,
                           // 2 = consumers skip the atomics (pure streaming rate of the ring), 4 = no L2 prefetch
};

// one (16 rows x group G) unit of the tile at shared address `rowaddr` (this lane's row, group 0): four LDS.32 at word
// offsets rotated per lane (the word rotation of the slot schedule is free in the address), then the 16 steps
template <bool GONLY, int G>
__device__ __forceinline__ void root_unit(const LaneConst& lc, const unsigned (&ldsoff)[4], unsigned rowaddr, int gq, unsigned hq) {
  constexpr int PL = GONLY ? 1 : 2;
  unsigned ww[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) ww[j] = lds_u32(rowaddr + (unsigned)(G * 32) + ldsoff[j]);
  accumulate16<GONLY, G * PL * kPlaneBytes>(lc, ww, gq, hq);
}

template <bool GONLY>
__global__ void __launch_bounds__(kRootThreads, 1)
hist_root_kernel(const __grid_constant__ CUtensorMap tm, HistArgs a, RootCfg c) {
  constexpr int PL = GONLY ? 1 : 2;
  constexpr int NCW = kRootConsumerWarps, R = kRootRows;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int nb = *a.build_count;
  if (nb <= 0) return;
  const unsigned T = a.build_prefix[nb];
  if (T == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g0 = blockIdx.y * a.ng_chunk;
  const int ng_here = min(a.ng_chunk, a.ngroups - g0);
  const bool has_tail = a.tw > 0 && blockIdx.y == gridDim.y - 1;
  if (a.rows_counter && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) atomicAdd(a.rows_counter, (unsigned long long)T);

  const unsigned smem_base = (unsigned)__cvta_generic_to_shared(smem_raw);
  const unsigned ring = (smem_base + c.ring_off + 127u) & ~127u;
  const unsigned bars = ring + (unsigned)c.S * c.stage_bytes;                 // full[S] then empty[S]
  const unsigned row_bytes = 32u * (unsigned)c.box_groups;
  const unsigned main_tile_bytes = (unsigned)R * row_bytes;
  constexpr unsigned kGradBytes = GONLY ? 4u : 8u;      // per row: the dense g, or the (g,h) pair
  const unsigned gp_off = main_tile_bytes, tail_tile_off = main_tile_bytes + (unsigned)R * kGradBytes;
  const unsigned ntiles = (T + R - 1) / R;
  const unsigned my_ntiles = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0u;   // tiles blockIdx.x + i * gridDim.x

  // zero the planes, init the barriers
  {
    const int main4 = ng_here * PL * kPlaneBytes / 16;
    int4* z = reinterpret_cast<int4*>(smem_raw);
    for (int i = threadIdx.x; i < main4; i += blockDim.x) z[i] = make_int4(0, 0, 0, 0);
    if (has_tail) {
      const int tail4 = PL * 256 * a.tw * c.trep * 4 / 16;
      int4* zt = reinterpret_cast<int4*>(smem_raw + c.tail_off);
      for (int i = threadIdx.x; i < tail4; i += blockDim.x) zt[i] = make_int4(0, 0, 0, 0);
    }
    if (threadIdx.x == 0) {
      for (int s = 0; s < c.S; ++s) { mbar_init(bars + 8u * s, 1); mbar_init(bars + 8u * (c.S + s), kTeamWarps); }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
  }
  __syncthreads();

  const int nid = a.build_nid[0];
  const size_t slot_entries = (size_t)a.ngroups * kGroupEntries + (size_t)256 * a.tw;
  GH64* out_slot = a.hist_pool + (size_t)a.hist_slot[nid] * slot_entries;
  GH64* out_main = out_slot + (size_t)g0 * kGroupEntries;
  GH64* out_tail = out_slot + (size_t)a.ngroups * kGroupEntries;

  if (warp >= NCW) {                                    // ---------------- producers: warp NCW + p issues tiles p, p + P, ...
    if (lane == 0) {
      const unsigned P = (c.flags & 8) ? 1u : (unsigned)kRootProducerWarps, pw = (unsigned)(warp - NCW);
      if (pw < P) {
        const unsigned tx = main_tile_bytes + (unsigned)R * kGradBytes + (has_tail ? (unsigned)R * (unsigned)a.tw : 0u);
        unsigned s = pw % (unsigned)c.S, round = pw / (unsigned)c.S;
        for (unsigned i = pw; i < my_ntiles; i += P) {
          if (round > 0) mbar_wait(bars + 8u * (c.S + s), (round - 1u) & 1u);
          const unsigned full = bars + 8u * s, dst = ring + s * c.stage_bytes;
          const unsigned t = blockIdx.x + i * gridDim.x;
          const unsigned row0 = t * (unsigned)R;
          mbar_expect_tx(full, tx);
          if ((c.flags & 1) && gridDim.y == 1) bulk_load_1d(dst, a.bins + (size_t)row0 * a.row_stride, main_tile_bytes, full);
          else tma_load_2d(dst, &tm, g0 * 32, (int)row0, full);
          if (GONLY) bulk_load_1d(dst + gp_off, a.gpos + row0, (unsigned)R * 4u, full);
          else bulk_load_1d(dst + gp_off, a.gpair + row0, (unsigned)R * 8u, full);
          if (has_tail) bulk_load_1d(dst + tail_tile_off, a.bins_tail + (size_t)row0 * a.tw, (unsigned)R * (unsigned)a.tw, full);
          const unsigned tp = t + 8u * gridDim.x;        // warm L2 eight tiles ahead of this CTA
          if (tp < ntiles && !(c.flags & 4)) tma_prefetch_2d(&tm, g0 * 32, (int)(tp * (unsigned)R));
          s += P; if (s >= (unsigned)c.S) { s -= (unsigned)c.S; ++round; }
        }
      }
    }
    return;
  }

  // ---------------- consumers
  const int team = warp / kTeamWarps, wit = warp % kTeamWarps;
  const float sg = a.scales[0], sh = a.scales[1];
  const LaneConst lc = make_lane_const(lane, smem_base);
  unsigned ldsoff[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { ldsoff[j] = 16u * (unsigned)(lane & 1) + 4u * (unsigned)((j + lc.qw) & 3); asm volatile("" : "+r"(ldsoff[j])); }
  TailConst tc;
  tc.tw = a.tw; tc.base_g = smem_base + c.tail_off; tc.hplane_bytes = 256u * (unsigned)a.tw * (unsigned)c.trep * 4u;
  tc.bin_stride = (unsigned)a.tw * (unsigned)c.trep * 4u;
  tc.rep_off = has_tail ? (unsigned)((lane / a.tw) % c.trep) * (unsigned)a.tw * 4u : 0u;
  const unsigned rowl = (unsigned)(wit << 4) + (unsigned)(lane >> 1);          // this lane's row inside a tile
  const unsigned tiles_per_window = (unsigned)a.window_rows / R;
  // GONLY: h == 1.0f for every row, so every valid row adds rint(1.0f * sh) to the node's H (hist_gather_kernel's GPAY rule)
  const unsigned hq_one = (unsigned)__float2int_rn(1.0f * sh);
  // (g_q, h_q) of tile row `row` from the stage's gradients; rows past T add nothing
  auto quant = [&](unsigned tile, unsigned row, bool valid, int& gq, unsigned& hq) {
    gq = 0; hq = 0;
    if constexpr (GONLY) {
      const float g = __uint_as_float(lds_u32(tile + gp_off + row * 4u));
      if (valid) { gq = __float2int_rn(g * sg); hq = hq_one; }
    } else {
      const uint2 gh = lds_v2(tile + gp_off + row * 8u);
      if (valid) { gq = __float2int_rn(__uint_as_float(gh.x) * sg); hq = (unsigned)__float2int_rn(__uint_as_float(gh.y) * sh); }
    }
  };
  long long accG = 0, accH = 0;
  unsigned i = (unsigned)team, s = (unsigned)team, ph = 0;                      // c.S >= kTeams (root_plan)
  for (unsigned wstart = 0;; wstart += tiles_per_window) {
    const unsigned wend = wstart + tiles_per_window < my_ntiles ? wstart + tiles_per_window : my_ntiles;
    while (i < wend) {
      mbar_wait(bars + 8u * s, ph);
      const unsigned tile = ring + s * c.stage_bytes;
      const unsigned row0 = (blockIdx.x + i * gridDim.x) * (unsigned)R;
      if (!(c.flags & 2)) {
        int gq; unsigned hq;
        quant(tile, rowl, row0 + rowl < T, gq, hq);
        if ((lane & 1) == 0) { accG += gq; accH += hq; }
        const unsigned rowaddr = tile + rowl * row_bytes;
        root_unit<GONLY, 0>(lc, ldsoff, rowaddr, gq, hq);
        if (ng_here > 1) root_unit<GONLY, 1>(lc, ldsoff, rowaddr, gq, hq);
        if (ng_here > 2) root_unit<GONLY, 2>(lc, ldsoff, rowaddr, gq, hq);
        if (has_tail) {
          const unsigned tu = ((unsigned)wit + i) & (unsigned)(kTeamWarps - 1);       // rotate the two 32-row tail units over the team
          if (tu < (unsigned)(R >> 5)) {
            const unsigned trow = (tu << 5) + (unsigned)lane;
            unsigned w0, w1 = 0;
            if (a.tw == 4) w0 = lds_u32(tile + tail_tile_off + trow * 4u);
            else { const uint2 ww = lds_v2(tile + tail_tile_off + trow * 8u); w0 = ww.x; w1 = ww.y; }
            int gqt; unsigned hqt;
            quant(tile, trow, row0 + trow < T, gqt, hqt);
            if (row0 + trow >= T) { w0 = 0; w1 = 0; }
            tail_accumulate<GONLY>(tc, lane, w0, w1, gqt, hqt);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + 8u * (c.S + s));
      i += kTeams; s += kTeams;
      if (s >= (unsigned)c.S) { s -= (unsigned)c.S; ph ^= 1u; }
    }
    if (wend == my_ntiles) break;
    named_bar_sync(1, NCW * 32);                          // overflow check: at most kWindowRows rows since the last one
    spill_main<PL>(reinterpret_cast<int*>(smem_raw), ng_here, out_main, false, threadIdx.x, NCW * 32);
    if (has_tail) spill_tail<PL>(reinterpret_cast<int*>(smem_raw + c.tail_off), a.tw, c.trep, out_tail, false, threadIdx.x, NCW * 32);
    named_bar_sync(1, NCW * 32);
  }
  named_bar_sync(1, NCW * 32);
  spill_main<PL>(reinterpret_cast<int*>(smem_raw), ng_here, out_main, true, threadIdx.x, NCW * 32);
  if (has_tail) spill_tail<PL>(reinterpret_cast<int*>(smem_raw + c.tail_off), a.tw, c.trep, out_tail, true, threadIdx.x, NCW * 32);
  if (a.accumulate_sum && blockIdx.y == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { accG += __shfl_xor_sync(0xffffffffu, accG, o); accH += __shfl_xor_sync(0xffffffffu, accH, o); }
    if (lane == 0 && (accG != 0 || accH != 0)) { red_global_s64(&a.node_sum[nid].g, accG); red_global_s64(&a.node_sum[nid].h, accH); }
  }
}

// ---------------------------------------------------------------------------------------------
// Deeper levels (and the fallback for the root): rows gathered by row id, register-staged.
// ---------------------------------------------------------------------------------------------
// one position per lane: row id, gradients (g alone with a G-only payload, else (g,h)) and the tail words
template <int TW, bool GPAY> struct Stage { unsigned id; typename std::conditional<GPAY, float, float2>::type gr; unsigned t0; };
template <bool GPAY> struct Stage<8, GPAY> { unsigned id; typename std::conditional<GPAY, float, float2>::type gr; unsigned t0, t1; };

// tail planes [bin][trep][tw] of the gather kernel: 32 KB (G + H, trep * tw = 16) fit next to three groups, 64 KB otherwise
__host__ __device__ constexpr int gather_tail_replicas(int ng) { return ng >= 3 ? 4 : 8; }
__host__ __device__ constexpr int gather_tail_bytes(int ng) { return ng >= 3 ? 32768 : 65536; }
// positions per super-tile of the gather kernel (see its lane mapping): 32, 32, 30 for NG = 1, 2, 3
__host__ __device__ constexpr int gather_super_rows(int ng) { return 32 / (2 * ng) * (2 * ng); }

// Rows of the build list per gather CTA: CTA x < ceff takes positions [x * chunk, min((x + 1) * chunk, T)), chunk a multiple of
// `sup`.  hist_reduce_kernel repeats it to find the CTAs of a node.
__device__ __forceinline__ void gather_split(unsigned T, unsigned C, unsigned sup, unsigned& ceff, unsigned& chunk) {
  ceff = (T + kMinRowsPerCta - 1) / kMinRowsPerCta;
  ceff = ceff < 1 ? 1 : (ceff > C ? C : ceff);
  chunk = (T + ceff - 1) / ceff;
  chunk = (chunk + sup - 1) / sup * sup;
}

// Final flush of a (CTA, node) segment of the gather kernel: the accumulators go to the segment's own partial slot with plain
// coalesced 16 B stores, one {g, h} int32 pair per slot entry, and the planes are zeroed for the next segment.  The tail
// replicas are summed first; a sum that does not fit 32 bits (only when several replicas sit near the spill threshold) goes
// to the pool with RED.ADD.64 instead, like a spill.
template <int TWC, int TREP>
__device__ __forceinline__ void flush_partials(int* smem, int* tsm, int ng_here, bool has_tail, int2* part_main, int2* part_tail, GH64* out_tail,
                                               int tid, int nthr) {
  constexpr int kHalf = kGroupEntries / 2;
#pragma unroll 1          // the gather kernel is register-bound: unrolled, this loop cost the one-group instantiations up to 38 registers
  for (int i = tid; i < ng_here * kHalf; i += nthr) {
    const int k = i / kHalf, e = (i - k * kHalf) * 2;
    int2* G = reinterpret_cast<int2*>(smem + k * 2 * kGroupEntries + e);
    int2* H = G + kHalf;
    const int2 g = *G, h = *H;
    *reinterpret_cast<int4*>(part_main + (size_t)k * kGroupEntries + e) = make_int4(g.x, h.x, g.y, h.y);
    *G = make_int2(0, 0); *H = make_int2(0, 0);
  }
  if (has_tail) {
    constexpr int kTailPlane = 256 * TWC * TREP;
    for (int e = tid; e < 256 * TWC; e += nthr) {
      const int bin = e / TWC, slot = e - bin * TWC;
      long long g = 0, h = 0;
#pragma unroll
      for (int r = 0; r < TREP; ++r) {
        int* t = tsm + (bin * TREP + r) * TWC + slot;
        g += t[0]; h += (unsigned)t[kTailPlane];
        t[0] = 0; t[kTailPlane] = 0;
      }
      if (g != (long long)(int)g) { red_global_s64(&out_tail[e].g, g); g = 0; }
      if (h != (long long)(unsigned)h) { red_global_s64(&out_tail[e].h, h); h = 0; }
      part_tail[e] = make_int2((int)g, (int)(unsigned)h);
    }
  }
}

// Lane mapping: a row's 32*NG contiguous bytes are fetched by 2*NG adjacent lanes of ONE LDG.128 instruction (the sectors of
// a row reach the L2 in one request, so DRAM serves them with whole 64 B bursts: requested by separate instructions a 96 B row
// cost ~2.6 bursts), i.e. 16 / 8 / 5 rows per instruction for NG = 1 / 2 / 3 (NG = 3 leaves lanes 30, 31 idle).  Lane (row q,
// chunk c) owns group c >> 1, half c & 1 and the slot rotation NG * q + (c >> 1): the <= 16 lanes that share a half have
// distinct rotations, so every ATOMS instruction is still bank-conflict free.
// GPAY (constant-hessian objectives): g alone by position from a.gpos; every valid row adds the constant h_q = rint(1.0f * sh)
// to the H plane, which is what the (g,h) path computes from h == 1.0f, so both planes come out bit-identical.
template <int NG, int TW, int NTHREADS, bool GPAY>       // TW: tail width this instantiation handles (0 = none, 4, 8)
__global__ void __launch_bounds__(NTHREADS, NG == 1 ? (TW ? 1 : 3) : 1) hist_gather_kernel(HistArgs a) {
  constexpr bool TAIL = TW != 0;
  constexpr int NWARPS = NTHREADS / 32;
  constexpr int LPR = 2 * NG, RPI = 32 / LPR, U = 2 * NG;                  // lanes per row, rows per instruction, units per super-tile
  constexpr int SUP = RPI * U;                                             // positions per super-tile: 32, 32, 30
  static_assert(SUP == gather_super_rows(NG), "hist_reduce_kernel splits the rows with gather_super_rows");
  static_assert(kWindowRowsSmall / (SUP * NWARPS) >= 1, "window too small");
  const unsigned iters_per_window = (unsigned)a.window_rows / (SUP * NWARPS);   // super-tiles per warp between overflow checks
  extern __shared__ __align__(16) int smem[];                              // per group: G[8192] then H[8192]; then the tail planes
  const int nb = *a.build_count;
  if (nb <= 0) return;
  const unsigned T = a.build_prefix[nb];
  if (T == 0) return;
  if (a.rows_counter && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) atomicAdd(a.rows_counter, (unsigned long long)T);
  unsigned ceff, chunk;
  gather_split(T, gridDim.x, SUP, ceff, chunk);
  if (blockIdx.x >= ceff) return;
  unsigned long long r0l = (unsigned long long)blockIdx.x * chunk;
  if (r0l >= T) return;
  unsigned r0 = (unsigned)r0l;
  unsigned r1 = (unsigned long long)r0 + chunk > T ? T : r0 + chunk;
  const int g0 = blockIdx.y * a.ng_chunk;
  const int ng_here = min(min(a.ng_chunk, NG), a.ngroups - g0);
  const bool has_tail = TAIL && a.tw > 0 && blockIdx.y == gridDim.y - 1;
  const float sg = a.scales[0], sh = a.scales[1];
  const unsigned smem_g = (unsigned)__cvta_generic_to_shared(smem);
  // gathered passes read the line-aligned copy of the rows; the contiguous pass (ridx == nullptr) the packed one
  const bool aligned = a.ridx != nullptr && a.bins_gather != nullptr;
  // tail bytes in the pad of the row's own aligned line: only 3 groups + an 8-wide tail have that layout, and the code must
  // not cost the other instantiations registers
  constexpr bool kLineTail = NG == 3 && TW == 8;
  const bool tail_line = kLineTail && aligned && a.tail_in_gather;
  const int64_t row_stride = aligned ? (int64_t)a.gather_stride : (int64_t)a.row_stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = lane / LPR, c = lane - q * LPR;                            // row inside a unit, 16 B chunk inside the row
  const bool lane_on = q < RPI && (c >> 1) < ng_here;                       // idle lanes add zeros to a slot rotation nobody else uses
  const int rot = q < RPI ? NG * q + (c >> 1) : 15;
  const LaneConst lc = make_lane_const_rot(rot, c & 1, smem_g + (unsigned)((q < RPI ? (c >> 1) : 0) * 2 * kPlaneBytes));
  const int rot_qw = rot >> 2, rot_qb8 = (rot & 3) * 8;
  const uint8_t* gbins = (aligned ? a.bins_gather : a.bins) + (int64_t)g0 * kSlots + c * 16;
  // tail planes [bin][trep][tw] behind the main planes; as many replicas as fit next to them
  constexpr int TWC = TAIL ? TW : 4;
  constexpr int trep = gather_tail_replicas(NG) < gather_tail_bytes(NG) / (2 * 256 * 4 * TWC) ? gather_tail_replicas(NG) : gather_tail_bytes(NG) / (2 * 256 * 4 * TWC);
  const unsigned tail_base_rep = smem_g + (unsigned)(NG * 2 * kPlaneBytes) + (unsigned)((lane / TWC) % trep) * (unsigned)TWC * 4u;

  {
    const int words4 = (NG * 2 * kPlaneBytes + (TAIL ? 2 * 256 * TWC * trep * 4 : 0)) / 16;
    for (int i = threadIdx.x; i < words4; i += NTHREADS) reinterpret_cast<int4*>(smem)[i] = make_int4(0, 0, 0, 0);
  }
  __syncthreads();

  int b = 0;   // first build node whose range contains r0
  { int lo = 0, hi = nb; while (lo < hi) { int mid = (lo + hi) >> 1; if (a.build_prefix[mid + 1] > r0) hi = mid; else lo = mid + 1; } b = lo; }

  const size_t slot_entries = (size_t)a.ngroups * kGroupEntries + (size_t)256 * a.tw;
  typedef Stage<TW, GPAY> StageT;
  const unsigned hq_one = (unsigned)__float2int_rn(1.0f * sh);              // GPAY: h_q of every row
  while (r0 < r1) {
    const unsigned nbeg = a.build_prefix[b], nend_node = a.build_prefix[b + 1];
    const unsigned nend = nend_node < r1 ? nend_node : r1;
    const int nid = a.build_nid[b];
    const unsigned seg = a.seg_begin[nid];
    GH64* out_slot = a.hist_pool + (size_t)a.hist_slot[nid] * slot_entries;
    GH64* out_main = out_slot + (size_t)g0 * kGroupEntries;
    GH64* out_tail = out_slot + (size_t)a.ngroups * kGroupEntries;
    int accG = 0; unsigned accH = 0;          // this lane's (g, h) since the last overflow check: <= iters_per_window rows, far from 32 bits
    const unsigned pa = seg + (r0 - nbeg), pb = seg + (nend - nbeg);
    const unsigned nsuper = (pb - pa + SUP - 1) / SUP;
    const unsigned iters = (nsuper + NWARPS - 1) / NWARPS;          // same for every warp: barriers stay aligned

    // Software pipeline per warp over super-tiles of SUP positions; it runs THROUGH the overflow-check barriers:
    //   row ids + gradients + tail bytes two super-tiles ahead (coalesced, one position per lane);
    //   bin chunks (one LDG.128 per lane and unit) one super-tile ahead, ROLLING: the register of unit k is refilled with
    //   unit k of the next super-tile right after it has been consumed (U loads in flight per lane at all times); on the
    //   aligned copy the tail bytes are requested right behind the bin chunks of the same lines (a request of its own two
    //   super-tiles earlier would fetch every line twice, and hang a dependent gather on the row-id load);
    //   conflict-free ATOMS pairs now.
    auto load_ids = [&](unsigned st) -> StageT {
      StageT s_; s_.id = 0xffffffffu; s_.gr = {}; s_.t0 = 0u;
      if constexpr (TW == 8) s_.t1 = 0u;
      unsigned p = pa + st * SUP + lane;
      if (lane < SUP && st < nsuper && p < pb) {
        s_.id = a.ridx ? __ldg(a.ridx + p) : p;
        if constexpr (GPAY) s_.gr = __uint_as_float(ldg_nc_u32(a.gpos + p)); else s_.gr = ldg_nc_f2(a.gpair + p);
        if (TAIL && has_tail && !tail_line) {
          if constexpr (TW == 8) { const uint2 v = ldg_nc_v2(a.bins_tail + (int64_t)s_.id * 8); s_.t0 = v.x; s_.t1 = v.y; }
          else if (a.tail_pos) s_.t0 = ldg_nc_u32(a.tail_pos + p);                  // tail bytes travel with the row ids (tw == 4)
          else s_.t0 = ldg_nc_u32(a.bins_tail + (int64_t)s_.id * 4);
        }
      }
      return s_;
    };
    auto load_unit = [&](unsigned ids, int k) -> uint4 {
      const unsigned rid = __shfl_sync(0xffffffffu, ids, q < RPI ? k * RPI + q : 0);
      return (lane_on && rid != 0xffffffffu) ? ldg_nc_v4(gbins + (int64_t)rid * row_stride) : make_uint4(0, 0, 0, 0);
    };
    auto load_line_tail = [&](StageT& s_) {
      if constexpr (TAIL) {
        if (tail_line && has_tail && s_.id != 0xffffffffu) {
          const uint8_t* t = a.bins_gather + (int64_t)s_.id * row_stride + a.ngroups * kSlots;
          if constexpr (TW == 8) { const uint2 v = ldg_nc_v2(t); s_.t0 = v.x; s_.t1 = v.y; } else s_.t0 = ldg_nc_u32(t);
        }
      }
    };
    StageT cur = load_ids(warp);
    StageT nxt = load_ids(warp + NWARPS);
    uint4 w[U];
#pragma unroll
    for (int k = 0; k < U; ++k) w[k] = load_unit(cur.id, k);
    load_line_tail(cur);
    for (unsigned it = 0; it < iters; ++it) {
      const unsigned s = warp + it * NWARPS;
      StageT nn = load_ids(s + 2 * NWARPS);
      const bool active = s < nsuper;
      int gq_l; unsigned hq_l;
      if constexpr (GPAY) { gq_l = __float2int_rn(cur.gr * sg); hq_l = cur.id != 0xffffffffu ? hq_one : 0u; }      // no row: adds nothing
      else { gq_l = __float2int_rn(cur.gr.x * sg); hq_l = (unsigned)__float2int_rn(cur.gr.y * sh); }
      accG += gq_l; accH += hq_l;
#pragma unroll
      for (int k = 0; k < U; ++k) {
        if (active) {
          int gq = __shfl_sync(0xffffffffu, gq_l, q < RPI ? k * RPI + q : 0);
          unsigned hq = __shfl_sync(0xffffffffu, hq_l, q < RPI ? k * RPI + q : 0);
          if (!lane_on) { gq = 0; hq = 0; }
          unsigned ww[4];
          rotate_words_bytes(rot_qw, rot_qb8, w[k], ww);
          accumulate16_pairs_prerotated<0>(lc.A, ww, gq, hq);
        }
        w[k] = load_unit(nxt.id, k);
      }
      if constexpr (TAIL) { if (active && has_tail) { unsigned t1 = 0; if constexpr (TW == 8) t1 = cur.t1; tail_accumulate_ct<TWC, trep>(tail_base_rep, lane, cur.t0, t1, gq_l, hq_l); } }
      load_line_tail(nxt);
      cur = nxt; nxt = nn;
      if ((it + 1) % iters_per_window == 0 && it + 1 < iters) {       // overflow check: at most kWindowRows rows since the last one
        if (a.accumulate_sum && blockIdx.y == 0) { flush_node_sum(a.node_sum + nid, accG, accH, lane); accG = 0; accH = 0; }
        __syncthreads();
        spill_main<2>(smem, ng_here, out_main, false, threadIdx.x, NTHREADS);
        if (has_tail) spill_tail<2>(smem + NG * 2 * kGroupEntries, TWC, trep, out_tail, false, threadIdx.x, NTHREADS);
        __syncthreads();
      }
    }
    __syncthreads();
    if (a.partials) {                        // segment b of CTA x: partial slot x + b (unique: a CTA's nodes are a contiguous run)
      int2* part = a.partials + (size_t)(blockIdx.x + b) * slot_entries;
      flush_partials<TWC, trep>(smem, smem + NG * 2 * kGroupEntries, ng_here, has_tail, part + (size_t)g0 * kGroupEntries,
                                part + (size_t)a.ngroups * kGroupEntries, out_tail, threadIdx.x, NTHREADS);
    } else {
      spill_main<2>(smem, ng_here, out_main, true, threadIdx.x, NTHREADS);
      if (has_tail) spill_tail<2>(smem + NG * 2 * kGroupEntries, TWC, trep, out_tail, true, threadIdx.x, NTHREADS);
    }
    __syncthreads();
    if (a.accumulate_sum && blockIdx.y == 0) flush_node_sum(a.node_sum + nid, accG, accH, lane);
    r0 = nend; ++b;
  }
}

// The partial slots of every built node added to its pool slot (which already holds the spills), in ascending CTA order.  Sums
// of integers: the same bits as the RED.ADD.64 flush in any order.  Node b's rows lie in the gather CTAs x_lo .. x_hi of a
// launch of C CTAs per group chunk, whose segments for it are partial slots x + b.  A thread takes two entries of a node.
__global__ void __launch_bounds__(256) hist_reduce_kernel(HistArgs a, unsigned C, unsigned sup) {
  const int nb = *a.build_count;
  if (nb <= 0) return;
  const unsigned T = a.build_prefix[nb];
  if (T == 0) return;
  unsigned ceff, chunk;
  gather_split(T, C, sup, ceff, chunk);
  const size_t slot_entries = (size_t)a.ngroups * kGroupEntries + (size_t)256 * a.tw;
  const size_t pairs = slot_entries / 2;
  for (size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x; item < (size_t)nb * pairs; item += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(item / pairs);
    const size_t p = item - (size_t)b * pairs;
    const unsigned nbeg = a.build_prefix[b], nend = a.build_prefix[b + 1];
    if (nbeg == nend) continue;
    const unsigned x_lo = nbeg / chunk, nseg = (nend - 1) / chunk - x_lo + 1;
    const int4* src = reinterpret_cast<const int4*>(a.partials + (size_t)(x_lo + b) * slot_entries) + p;
    long long g0 = 0, h0 = 0, g1 = 0, h1 = 0;
    auto add = [&](const int4& v) { g0 += v.x; h0 += (unsigned)v.y; g1 += v.z; h1 += (unsigned)v.w; };
    unsigned s = 0;
    for (; s + 8 <= nseg; s += 8) {                     // eight loads in flight per thread
      int4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __ldcs(src + (size_t)(s + j) * pairs);
#pragma unroll
      for (int j = 0; j < 8; ++j) add(v[j]);
    }
    for (; s < nseg; ++s) add(__ldcs(src + (size_t)s * pairs));
    longlong2* o = reinterpret_cast<longlong2*>(a.hist_pool + (size_t)a.hist_slot[a.build_nid[b]] * slot_entries + 2 * p);
    longlong2 e0 = o[0], e1 = o[1];
    e0.x += g0; e0.y += h0; e1.x += g1; e1.y += h1;
    o[0] = e0; o[1] = e1;
  }
}

// ---------------------------------------------------------------------------------------------
// host side: kernel selection, shared-memory plan of the root kernel, tensor maps
// ---------------------------------------------------------------------------------------------
static thread_local const char* g_last_kernel = "none";
const char* hist_last_kernel() { return g_last_kernel; }

static int chunks_for(int ngroups) { return (ngroups + 2) / 3; }
static int groups_per_chunk(int ngroups) { const int nc = chunks_for(ngroups); return (ngroups + nc - 1) / nc; }
// CTAs per group chunk of hist_gather_kernel
static int gather_grid_x(int ngroups, int tw, int num_sms) {
  const int nchunks = chunks_for(ngroups);
  const int per_sm = groups_per_chunk(ngroups) > 1 ? 1 : (tw ? 1 : 3);   // one group: 64 KB of planes (+ 64 KB of replicated tail planes) per CTA
  return (num_sms * per_sm + nchunks - 1) / nchunks;
}
size_t hist_partial_entries(int ngroups, int tw, int num_sms, int max_build) {
  return ((size_t)gather_grid_x(ngroups, tw, num_sms) + (size_t)max_build) * hist_slot_entries(ngroups, tw);
}

// Shared-memory plan of hist_root_kernel; returns false when the ring next to the planes would be too shallow to keep
// every team busy (3 groups of G+H planes = 192 KB: that shape uses the gather kernel for its root pass).
static bool root_plan(int ngc, int tw, bool gonly, RootCfg* c) {
  const int PL = gonly ? 1 : 2;
  const unsigned main_b = (unsigned)ngc * PL * kPlaneBytes;
  const unsigned avail = kMaxSmem - 128 /* alignment slack */ - 2 * 8 * 16 /* barriers */;
  // a stage: the tile's bins, its gradients (dense g: 4 B per row, (g,h): 8 B) and its tail bytes.  kRootRows * each of these is
  // a multiple of 256 B, so every bulk copy's size and shared-memory address stay 16 B (and the TMA boxes 128 B) aligned
  const unsigned stage = (unsigned)kRootRows * (32u * ngc + (gonly ? 4u : 8u) + tw);
  int trep = tw ? 32 / tw : 0;
  unsigned tail_b = (unsigned)PL * 256u * tw * trep * 4u;
  if (tw && main_b + tail_b + kTeams * stage > avail) { trep = 1; tail_b = (unsigned)PL * 256u * tw * 4u; }
  if (main_b + tail_b + kTeams * stage > avail) return false;
  int S = (int)((avail - main_b - tail_b) / stage);
  int smax = 16;
  if (const char* e = getenv("B200XGB_ROOT_S")) smax = atoi(e);
  if (S > smax) S = smax;
  // a ring stage must always be refilled by the SAME producer thread (a parity wait may only ever be one phase ahead of its
  // barrier, which a single thread's program order guarantees): tile i -> producer i % P -> stage i % S needs S % P == 0
  // ... and likewise always consumed by the SAME team (tile i -> team i % kTeams): S must be a multiple of both
  constexpr int kStageQuantum = kTeams % kRootProducerWarps == 0 ? kTeams : kTeams * kRootProducerWarps;
  S -= S % kStageQuantum;
  if (S < kTeams) return false;
  c->S = S; c->trep = trep; c->box_groups = ngc; c->tail_off = main_b; c->ring_off = main_b + tail_b; c->stage_bytes = stage;
  c->total = main_b + tail_b + 128 + (unsigned)S * stage + 2 * 8 * (unsigned)S;
  c->flags = 0;
  if (const char* f = getenv("B200XGB_ROOT_FLAGS")) c->flags = atoi(f);
  return true;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); p = nullptr; }
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// tensor map of the main block [n][row_stride] uint8 with box {32 * box_groups, R}; cached per (pointer, shape, box)
static bool get_tensor_map(const uint8_t* bins, int64_t n, int row_stride, int box_groups, int R, CUtensorMap* out) {
  typedef std::tuple<const void*, int64_t, int, int, int> Key;
  static std::map<Key, CUtensorMap> cache; static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  const Key key(bins, n, row_stride, box_groups, R);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return true; }
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  CUtensorMap tm;
  const cuuint64_t dims[2] = {(cuuint64_t)row_stride, (cuuint64_t)n};
  const cuuint64_t strides[1] = {(cuuint64_t)row_stride};
  const cuuint32_t box[2] = {(cuuint32_t)(32 * box_groups), (cuuint32_t)R};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(bins), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  if (cache.size() > 64) cache.clear();
  cache[key] = tm; *out = tm;
  return true;
}

template <int NG, int TW, int NT> static void set_gather_attr() {
  const int smem = NG * 2 * kPlaneBytes + (TW ? gather_tail_bytes(NG) : 0);
  CUDA_OK(cudaFuncSetAttribute(hist_gather_kernel<NG, TW, NT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CUDA_OK(cudaFuncSetAttribute(hist_gather_kernel<NG, TW, NT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}

void hist_configure() {
  static bool configured = false;
  if (configured) return;
  set_gather_attr<1, 0, 256>(); set_gather_attr<1, 4, 256>(); set_gather_attr<1, 8, 256>();
  set_gather_attr<2, 0, 768>(); set_gather_attr<2, 4, 768>(); set_gather_attr<2, 8, 768>();
  set_gather_attr<3, 0, 768>(); set_gather_attr<3, 4, 768>(); set_gather_attr<3, 8, 768>();
  CUDA_OK(cudaFuncSetAttribute(hist_root_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  CUDA_OK(cudaFuncSetAttribute(hist_root_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  configured = true;
}

template <int NG, int NT, bool GPAY>
static void launch_gather_tw(const HistArgs& a, int gx, int nchunks, cudaStream_t stream) {
  const int smem = NG * 2 * kPlaneBytes + (a.tw ? gather_tail_bytes(NG) : 0);
  if (a.tw == 0) hist_gather_kernel<NG, 0, NT, GPAY><<<dim3(gx, nchunks), NT, smem, stream>>>(a);
  else if (a.tw == 4) hist_gather_kernel<NG, 4, NT, GPAY><<<dim3(gx, nchunks), NT, smem, stream>>>(a);
  else hist_gather_kernel<NG, 8, NT, GPAY><<<dim3(gx, nchunks), NT, smem, stream>>>(a);
}
template <int NG, int NT>
static void launch_gather(const HistArgs& a, int gx, int nchunks, cudaStream_t stream) {
  if (a.gpos) launch_gather_tw<NG, NT, true>(a, gx, nchunks, stream); else launch_gather_tw<NG, NT, false>(a, gx, nchunks, stream);
}

void launch_hist_build(const HistArgs& a_in, int num_sms, cudaStream_t stream) {
  HistArgs a = a_in;
  const int nchunks = chunks_for(a.ngroups);
  a.ng_chunk = groups_per_chunk(a.ngroups);
  static const bool no_tma = getenv("B200XGB_NO_TMA") != nullptr;
  // the root kernel streams (g,h) pairs, or in its G-only mode the dense g; the contiguous pass of a G-only payload that needs
  // the H plane too (gpos without g_only) runs in hist_gather_kernel
  const bool gonly = a.g_only != 0;
  B200_CHECK(!gonly || a.gpos != nullptr, "hist: the G-only root pass reads the dense g (gpos)");
  if (a.ridx == nullptr && !no_tma && !a.force_gather && (a.gpos == nullptr || gonly)) {
    RootCfg c; CUtensorMap tm;
    if (root_plan(a.ng_chunk, a.tw, gonly, &c) && get_tensor_map(a.bins, a.n, a.row_stride, c.box_groups, kRootRows, &tm)) {
      const int gx = num_sms / nchunks > 0 ? num_sms / nchunks : 1;
      if (gonly) hist_root_kernel<true><<<dim3(gx, nchunks), kRootThreads, c.total, stream>>>(tm, a, c);
      else hist_root_kernel<false><<<dim3(gx, nchunks), kRootThreads, c.total, stream>>>(tm, a, c);
      g_last_kernel = gonly ? "hist_root_kernel<GONLY>" : "hist_root_kernel<GH>";
      ++g_kernel_launches;
      CUDA_OK(cudaGetLastError());
      return;
    }
  }
  B200_CHECK(!a.g_only || a.ridx == nullptr, "hist: G-only accumulation is a root-pass mode");
  B200_CHECK(!a.g_only, "hist: the G-only root pass needs the TMA kernel (tensor-map creation failed or B200XGB_NO_TMA is set)");
  // the gathered passes end each (CTA, node) segment with plain stores into its partial slot and one reduce launch sums them;
  // B200XGB_HIST_RED_FLUSH=1 keeps the RED.ADD.64 flush into the pool (the A/B reference of the tests)
  static const bool red_flush = getenv("B200XGB_HIST_RED_FLUSH") != nullptr;
  if (red_flush) a.partials = nullptr;
  else B200_CHECK(a.partials != nullptr, "hist: the gathered passes need the builder's partial histograms");
  const int ng = a.ng_chunk;
  const int gx = gather_grid_x(a.ngroups, a.tw, num_sms);
  if (ng == 1) launch_gather<1, 256>(a, gx, nchunks, stream);
  else if (ng == 2) launch_gather<2, 768>(a, gx, nchunks, stream);
  else launch_gather<3, 768>(a, gx, nchunks, stream);
  g_last_kernel = "hist_gather_kernel";
  ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  if (a.partials) {
    hist_reduce_kernel<<<num_sms * 8, 256, 0, stream>>>(a, (unsigned)gx, (unsigned)gather_super_rows(ng));
    ++g_kernel_launches;
    CUDA_OK(cudaGetLastError());
  }
}

}  // namespace b200
