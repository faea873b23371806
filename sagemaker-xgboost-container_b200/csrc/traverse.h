// traverse.h -- the predictor's walk of one row through one tree on the raw float matrix (misc.cu predict_kernel), shared with
// the tree refresh (refresh.cu) so that a refreshed node sees exactly the rows the predictor sends through it.
#pragma once
#include "misc.h"

namespace b200 {

// The leaf a row reaches in `nodes`, where load(f) is the row's feature f (NaN when missing): x < cond goes left, a missing
// value follows default_left.
template <typename Load>
__device__ __forceinline__ int tree_leaf_by(const DevNode* nodes, Load load, DevNode* leaf) {
  int nid = 0;
  DevNode nd = nodes[0];
  while (nd.left != -1) {
    const float v = load(nd.fidx_dl & 0x7fffffffu);
    if (isnan(v)) nid = (nd.fidx_dl >> 31) ? nd.left : nd.right;
    else nid = v < nd.cond ? nd.left : nd.right;
    nd = nodes[nid];
  }
  *leaf = nd;
  return nid;
}

// The leaf row x (F features) reaches in `nodes`: x < cond goes left, a missing value (NaN, or a feature the matrix lacks)
// follows default_left.
__device__ __forceinline__ int tree_leaf(const DevNode* nodes, const float* x, int F, DevNode* leaf) {
  return tree_leaf_by(nodes, [&](unsigned f) { return f < (unsigned)F ? __ldg(x + f) : __int_as_float(0x7fc00000); }, leaf);
}

}  // namespace b200
