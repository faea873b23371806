// dart.cu -- booster=dart: the margins of a weighted list of trees, walked once per row on the raw feature matrix.
// Serves the DART round (booster.cu update_one_iter: the margin without the dropped trees for the gradients, the new weights
// of the dropped trees into the training cache), the catch-up of prediction caches after weights changed, and prediction of
// a dart model.  The arithmetic is defined so that the oracle can restate it bit for bit: for each listed tree j in list
// order, with its leaf value v on the row and its class column c,
//   m_drop[c] = m_drop[c] - fl(coef_drop[j] * v)   (m_drop starts as a copy of m_full)
//   m_full[c] = m_full[c] + fl(coef_full[j] * v)
// every product and sum rounded to nearest (no contraction into an FMA).
#include "engine.h"
#include "misc.h"

namespace b200 {

__device__ __forceinline__ float dart_leaf(const DevNode* nodes, const float* x, int F) {
  DevNode nd = nodes[0];
  while (nd.left != -1) {
    const unsigned f = nd.fidx_dl & 0x7fffffffu;
    const float v = f < (unsigned)F ? __ldg(x + f) : __int_as_float(0x7fc00000);
    const int nid = isnan(v) ? ((nd.fidx_dl >> 31) ? nd.left : nd.right) : (v < nd.cond ? nd.left : nd.right);
    nd = nodes[nid];
  }
  return nd.cond;
}

// one thread per row; K == 1 keeps both margins in registers, K > 1 updates the row's class columns in place
template <bool DROP>
__global__ void __launch_bounds__(256) dart_margin_kernel(DartArgs a) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n) return;
  const float* x = a.X + r * a.F;
  if (a.K == 1) {
    float mf = a.m_full[r], md = mf;
    for (int j = 0; j < a.ntrees; ++j) {
      const float v = dart_leaf(a.nodes + a.tree_offset[a.trees[j]], x, a.F);
      if (DROP) md = __fadd_rn(md, -__fmul_rn(a.coef_drop[j], v));
      mf = __fadd_rn(mf, __fmul_rn(a.coef_full[j], v));
    }
    a.m_full[r] = mf;
    if (DROP) a.m_drop[r] = md;
    return;
  }
  float* mf = a.m_full + r * a.K;
  float* md = DROP ? a.m_drop + r * a.K : nullptr;
  if (DROP) for (int k = 0; k < a.K; ++k) md[k] = mf[k];
  for (int j = 0; j < a.ntrees; ++j) {
    const float v = dart_leaf(a.nodes + a.tree_offset[a.trees[j]], x, a.F);
    const int c = a.tree_info[a.trees[j]];
    if (DROP) md[c] = __fadd_rn(md[c], -__fmul_rn(a.coef_drop[j], v));
    mf[c] = __fadd_rn(mf[c], __fmul_rn(a.coef_full[j], v));
  }
}

void launch_dart_margin(const DartArgs& a, cudaStream_t s) {
  if (a.n == 0 || a.ntrees == 0) return;
  const unsigned grid = (unsigned)((a.n + 255) / 256);
  if (a.m_drop) dart_margin_kernel<true><<<grid, 256, 0, s>>>(a);
  else dart_margin_kernel<false><<<grid, 256, 0, s>>>(a);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
