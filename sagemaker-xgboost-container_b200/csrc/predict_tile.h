// predict_tile.h -- what the two tiled predictors share: misc.cu predict_tiled_kernel (rows of floats) and predict_bins.cu
// predict_bins_tiled_kernel (rows of bin codes) stage a chunk of trees in shared memory the same way and walk a staged row
// through it the same way; they differ in how a tile of rows is staged and how a split reads its row.
#pragma once
#include "misc.h"

namespace b200 {

struct PNode { float cond; unsigned w; };            // w = left child (16 bit, 0xffff = leaf) | feature << 16 | default_left << 31

// PNode::w keeps 15 bits of feature id: the plans tile only rows of at most kPredictMaxPitch features
static_assert(kPredictMaxPitch <= 0x7fff + 1, "the tiled predictor's feature field has 15 bits");

// Trees [tree_lo, tree_hi) packed at the head of psm (predict_plan.h predict_chunk_head): their node offsets, then 8 B per
// node.  Returns the first byte behind the nodes, where the caller stages its rows; the caller synchronises before reading.
__device__ __forceinline__ unsigned char* stage_tree_chunk(const PredictArgs& a, int tree_lo, int tree_hi, unsigned char* psm, int** s_toff_out,
                                                           PNode** s_nodes_out) {
  const int nt_chunk = tree_hi - tree_lo;
  int* s_toff = reinterpret_cast<int*>(psm);                                   // [nt_chunk + 1] node offsets inside s_nodes
  PNode* s_nodes = reinterpret_cast<PNode*>(psm + (((size_t)(nt_chunk + 1) * 4 + 15) & ~(size_t)15));
  __shared__ int s_total;
  if (threadIdx.x == 0) {
    int off = 0;
    for (int t = 0; t < nt_chunk; ++t) { s_toff[t] = off; off += (int)(a.tree_offset[tree_lo + t + 1] - a.tree_offset[tree_lo + t]); }
    s_toff[nt_chunk] = off; s_total = off;
  }
  __syncthreads();
  for (int t = 0; t < nt_chunk; ++t) {
    const DevNode* src = a.nodes + a.tree_offset[tree_lo + t];
    const int cnt = s_toff[t + 1] - s_toff[t];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const DevNode d = src[i];
      PNode p; p.cond = d.cond;
      p.w = (d.left < 0 ? 0xffffu : (unsigned)d.left) | ((d.fidx_dl & 0x7fffu) << 16) | (d.fidx_dl & 0x80000000u);
      s_nodes[s_toff[t] + i] = p;
    }
  }
  *s_toff_out = s_toff; *s_nodes_out = s_nodes;
  return reinterpret_cast<unsigned char*>(s_nodes + s_total);
}

// Row r through the chunk's trees: go_left(node) decides a split on the staged row.  Leaves are summed in fp32 in tree
// order (K == 1; the reference's sequential sum) or added to their class's margin; LEAF_OUT writes the leaf ids instead.
template <bool LEAF_OUT, typename GoLeft>
__device__ __forceinline__ void predict_staged_row(const PredictArgs& a, const PNode* s_nodes, const int* s_toff, int nt_chunk, int tree_lo, int64_t r,
                                                   GoLeft go_left) {
  const int K = a.K, nt_all = a.tree_end - a.tree_begin;
  float acc = (!LEAF_OUT && K == 1) ? a.margin[r] : 0.f;
  auto step = [&](const PNode* tn, int& nid, PNode& nd) {
    const int left = (int)(nd.w & 0xffffu);
    nid = go_left(nd) ? left : left + 1;                                      // children are allocated as adjacent pairs
    nd = tn[nid];
  };
  auto emit = [&](int t, int nid, const PNode& nd) {
    if (LEAF_OUT) a.leaf[r * nt_all + (tree_lo - a.tree_begin) + t] = nid;
    else if (K == 1) acc += nd.cond;
    else a.margin[r * K + a.tree_info[tree_lo + t]] += nd.cond;
  };
  int t = 0;
  for (; t + 4 <= nt_chunk; t += 4) {                                         // four independent traversals in flight hide the LDS latency
    const PNode* tn[4]; int nid[4]; PNode nd[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { tn[j] = s_nodes + s_toff[t + j]; nid[j] = 0; nd[j] = tn[j][0]; }
    bool any = true;
    while (any) {
      any = false;
#pragma unroll
      for (int j = 0; j < 4; ++j) if ((nd[j].w & 0xffffu) != 0xffffu) { step(tn[j], nid[j], nd[j]); any = true; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) emit(t + j, nid[j], nd[j]);
  }
  for (; t < nt_chunk; ++t) {
    const PNode* tn = s_nodes + s_toff[t];
    int nid = 0; PNode nd = tn[0];
    while ((nd.w & 0xffffu) != 0xffffu) step(tn, nid, nd);
    emit(t, nid, nd);
  }
  if (!LEAF_OUT && K == 1) a.margin[r] = acc;
}

}  // namespace b200
