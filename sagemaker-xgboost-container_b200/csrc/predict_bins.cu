// predict_bins.cu -- the predictor on a binned matrix (a QuantileDMatrix keeps no float copy of its features).
// Each value stands at the lower edge of its bin: min_vals[f] for bin 0, else cut_vals[ptr[f] + b - 1].  A split `x < cond`
// becomes `b < t`, t = the number of the feature's lower edges below cond, and a missing value (code 255 under has_missing)
// takes the default direction.  For cond a cut value of the matrix, or its min_vals[f], every value of a bin lies on the
// same side of cond as the bin's lower edge, so the branch is the float predictor's (DESIGN.md "QuantileDMatrix").
// The kernels mirror misc.cu's predictor: a thread-per-row kernel (on the column-major copy, coalesced across the warp) and
// a tiled kernel that stages rows of bin codes in shared memory; leaves are summed per row in tree order in fp32.
#include <algorithm>
#include <cstdlib>
#include "misc.h"
#include "predict_tile.h"

namespace b200 {

// t for every split node: a binary search over the feature's lower edges (min, cut[0], ..., cut[nb - 2])
__global__ void __launch_bounds__(256) bin_thresholds_kernel(const DevNode* nodes, size_t count, const int* cut_ptrs, const float* cut_vals,
                                                             const float* min_vals, int F, DevNode* out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
    DevNode d = nodes[i];
    if (d.left != -1) {
      const unsigned f = d.fidx_dl & 0x7fffffffu, dl = d.fidx_dl & 0x80000000u;
      int t;
      if (f >= (unsigned)F) { t = dl ? 512 : 0; d.fidx_dl = dl; }       // a feature the matrix lacks reads as missing
      else {
        const float* c = cut_vals + cut_ptrs[f];
        const int nb = cut_ptrs[f + 1] - cut_ptrs[f];
        if (!(min_vals[f] < d.cond)) t = 0;
        else {                                                         // 1 + #{j < nb - 1 : c[j] < cond}
          int lo = 0, hi = nb - 1;
          while (lo < hi) { const int mid = (lo + hi) >> 1; if (c[mid] < d.cond) lo = mid + 1; else hi = mid; }
          t = 1 + lo;
        }
      }
      d.cond = __int_as_float(t);
    }
    out[i] = d;
  }
}

__device__ __forceinline__ bool bin_go_left(unsigned b, const DevNode& nd, bool has_missing) {
  if (has_missing && b == (unsigned)kMissingBin) return (nd.fidx_dl >> 31) != 0;
  return (int)b < __float_as_int(nd.cond);
}

// one thread per row, reading bins_col[f][r]
__global__ void __launch_bounds__(256) predict_bins_kernel(PredictArgs a, const uint8_t* __restrict__ cols, int has_missing) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n) return;
  const int nt = a.tree_end - a.tree_begin;
  float acc = (a.K == 1 && a.margin) ? a.margin[r] : 0.f;
  for (int t = a.tree_begin; t < a.tree_end; ++t) {
    const DevNode* tn = a.nodes + a.tree_offset[t];
    int nid = 0;
    DevNode nd = tn[0];
    while (nd.left != -1) {
      const unsigned f = nd.fidx_dl & 0x7fffffffu;
      nid = bin_go_left(__ldg(cols + (int64_t)f * a.n + r), nd, has_missing != 0) ? nd.left : nd.right;
      nd = tn[nid];
    }
    if (a.margin) { if (a.K == 1) acc += nd.cond; else a.margin[r * a.K + a.tree_info[t]] += nd.cond; }
    if (a.leaf) a.leaf[r * nt + (t - a.tree_begin)] = nid;
  }
  if (a.K == 1 && a.margin) a.margin[r] = acc;
}

// Rows of bin codes, row r's main bytes at src + r * src_stride and its tail bytes at tail + r * tw (or, with tail_in_src, right
// behind the main bytes in src), staged in shared memory as pitch 4-byte words: byte f of a staged row is feature f.
struct BinRows { const uint8_t* src; const uint8_t* tail; int src_stride, main_words, tail_words, tail_in_src; };

template <bool HAS_MISSING, bool LEAF_OUT>
__global__ void __launch_bounds__(1024) predict_bins_tiled_kernel(PredictArgs a, BinRows br, int tree_lo, int tree_hi, int pitch, int rows_per_tile,
                                                                  int64_t num_tiles) {
  extern __shared__ __align__(16) unsigned char psm[];
  int* s_toff; PNode* s_nodes;                                                  // a split's cond holds its threshold t as int bits
  unsigned* s_x = reinterpret_cast<unsigned*>(stage_tree_chunk(a, tree_lo, tree_hi, psm, &s_toff, &s_nodes));
  const int nt_chunk = tree_hi - tree_lo;
  const int rw = br.main_words + br.tail_words;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t r0 = tile * rows_per_tile;
    const int rows = (int)((a.n - r0 < rows_per_tile) ? a.n - r0 : rows_per_tile);
    __syncthreads();                                                            // trees staged / previous tile consumed
    for (int i = threadIdx.x; i < rows * rw; i += blockDim.x) {
      const int r = i / rw, c = i - r * rw;
      const int64_t row = r0 + r;
      unsigned v;
      if (c < br.main_words || br.tail_in_src) v = __ldg(reinterpret_cast<const unsigned*>(br.src + row * br.src_stride) + c);
      else v = __ldg(reinterpret_cast<const unsigned*>(br.tail + row * (br.tail_words * 4)) + (c - br.main_words));
      s_x[r * pitch + c] = v;
    }
    __syncthreads();
    for (int rl = threadIdx.x; rl < rows; rl += blockDim.x) {
      const uint8_t* x = reinterpret_cast<const uint8_t*>(s_x + rl * pitch);
      predict_staged_row<LEAF_OUT>(a, s_nodes, s_toff, nt_chunk, tree_lo, r0 + rl, [&](const PNode& nd) {
        const unsigned b = x[(nd.w >> 16) & 0x7fffu];
        bool go_left = (int)b < __float_as_int(nd.cond);
        if (HAS_MISSING) { if (b == (unsigned)kMissingBin) go_left = (nd.w >> 31) != 0; }
        return go_left;
      });
    }
  }
}

void launch_bin_thresholds(const DevNode* nodes, size_t count, const int* cut_ptrs, const float* cut_vals, const float* min_vals, int F,
                           DevNode* out, cudaStream_t s) {
  if (count == 0) return;
  const int grid = (int)std::min<size_t>((count + 255) / 256, (size_t)engine_num_sms() * 8);
  bin_thresholds_kernel<<<grid, 256, 0, s>>>(nodes, count, cut_ptrs, cut_vals, min_vals, F, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

// B200XGB_PREDICT_LEGACY (read once per process) forces thread-per-row, as for the float predictor
PredictPlan plan_for_bins(const PredictArgs& a, const BinnedMatrix& m) {
  static const bool legacy = getenv("B200XGB_PREDICT_LEGACY") != nullptr;
  return plan_predict_bins(a.h_tree_offset, a.tree_begin, a.tree_end, m.ngroups * kSlots + m.tw, a.children_adjacent != 0, legacy);
}

void launch_predict_bins(const PredictArgs& a, const BinnedMatrix& m, cudaStream_t s) {
  if (a.n == 0 || a.tree_end <= a.tree_begin) return;
  const PredictPlan plan = plan_for_bins(a, m);
  if (plan.kernel == PredictKernel::kTiled) {
    static bool attr = false;
    if (!attr) {
      CUDA_OK(cudaFuncSetAttribute(predict_bins_tiled_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPredictSmem));
      CUDA_OK(cudaFuncSetAttribute(predict_bins_tiled_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPredictSmem));
      CUDA_OK(cudaFuncSetAttribute(predict_bins_tiled_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPredictSmem));
      CUDA_OK(cudaFuncSetAttribute(predict_bins_tiled_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPredictSmem));
      attr = true;
    }
    BinRows br{};
    const int W = m.ngroups * kSlots;
    br.main_words = W / 4; br.tail_words = m.tw / 4; br.tail = m.bins_tail;
    if (m.bins_gather != m.bins) { br.src = m.bins_gather; br.src_stride = m.gather_stride; br.tail_in_src = m.tail_in_gather; }   // the aligned 128 B copy
    else { br.src = m.bins; br.src_stride = W; br.tail_in_src = 0; }
    for (const PredictChunk& ch : plan.chunks) {
      const int rows = ch.rows, threads = ch.threads;
      const int64_t tiles = (a.n + rows - 1) / rows;
      const int grid = (int)std::min<int64_t>(tiles, engine_num_sms() * (threads == 1024 ? 1 : 2048 / threads));
      if (a.leaf) { if (m.has_missing) predict_bins_tiled_kernel<true, true><<<grid, threads, ch.smem, s>>>(a, br, ch.tree_lo, ch.tree_hi, plan.pitch, rows, tiles);
                    else predict_bins_tiled_kernel<false, true><<<grid, threads, ch.smem, s>>>(a, br, ch.tree_lo, ch.tree_hi, plan.pitch, rows, tiles); }
      else { if (m.has_missing) predict_bins_tiled_kernel<true, false><<<grid, threads, ch.smem, s>>>(a, br, ch.tree_lo, ch.tree_hi, plan.pitch, rows, tiles);
             else predict_bins_tiled_kernel<false, false><<<grid, threads, ch.smem, s>>>(a, br, ch.tree_lo, ch.tree_hi, plan.pitch, rows, tiles); }
      ++g_kernel_launches; CUDA_OK(cudaGetLastError());
    }
    return;
  }
  predict_bins_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, s>>>(a, m.bins_col, m.has_missing); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
