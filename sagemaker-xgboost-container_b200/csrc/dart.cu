// dart.cu -- booster=dart: the margins of a weighted list of trees, walked once per row on the raw feature matrix.
// Serves the DART round (booster.cu update_one_iter: the margin without the dropped trees for the gradients, the new weights
// of the dropped trees into the training cache), the catch-up of prediction caches after weights changed, and prediction of
// a dart model.  The arithmetic is defined so that the oracle can restate it bit for bit: for each listed tree j in list
// order, with its leaf value v on the row and its class column c,
//   m_drop[c] = m_drop[c] - fl(coef_drop[j] * v)   (m_drop starts as a copy of m_full)
//   m_full[c] = m_full[c] + fl(coef_full[j] * v)
// every product and sum rounded to nearest (no contraction into an FMA).
#include "engine.h"
#include "inplace.h"
#include "misc.h"
#include "traverse.h"

namespace b200 {

// the leaf value row r of src reaches in `nodes` (src: inplace.h, the DMatrix's matrix or an in-place input)
template <class Src>
__device__ __forceinline__ float dart_leaf(const DevNode* nodes, const Src& src, int64_t r) {
  DevNode nd;
  tree_leaf_by(nodes, [&](unsigned f) { return src.at(r, (int)f); }, &nd);
  return nd.cond;
}

// one thread per row; K == 1 keeps both margins in registers, K > 1 updates the row's class columns in place
template <bool DROP, class Src>
__global__ void __launch_bounds__(256) dart_margin_kernel(DartArgs a, Src x) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n) return;
  if (a.K == 1) {
    float mf = a.m_full[r], md = mf;
    for (int j = 0; j < a.ntrees; ++j) {
      const float v = dart_leaf(a.nodes + a.tree_offset[a.trees[j]], x, r);
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
    const float v = dart_leaf(a.nodes + a.tree_offset[a.trees[j]], x, r);
    const int c = a.tree_info[a.trees[j]];
    if (DROP) md[c] = __fadd_rn(md[c], -__fmul_rn(a.coef_drop[j], v));
    mf[c] = __fadd_rn(mf[c], __fmul_rn(a.coef_full[j], v));
  }
}

void launch_dart_margin(const DartArgs& a, cudaStream_t s) {
  if (a.n == 0 || a.ntrees == 0) return;
  const unsigned grid = (unsigned)((a.n + 255) / 256);
  const RowsF32 x{a.X, a.F};
  if (a.m_drop) dart_margin_kernel<true><<<grid, 256, 0, s>>>(a, x);
  else dart_margin_kernel<false><<<grid, 256, 0, s>>>(a, x);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

void launch_dart_margin_inplace(const DartArgs& a, const InputDesc& d, cudaStream_t s) {
  B200_CHECK(a.m_drop == nullptr && a.n == d.n, "launch_dart_margin_inplace: the full margin of the input's rows only");
  if (a.n == 0 || a.ntrees == 0) return;
  const unsigned grid = (unsigned)((a.n + 255) / 256);
  if (d.indptr) dart_margin_kernel<false><<<grid, 256, 0, s>>>(a, CsrSrc{d});
  else if (d.type == kInF32) dart_margin_kernel<false><<<grid, 256, 0, s>>>(a, StridedSrc<kInF32>{d});
  else if (d.type == kInF64) dart_margin_kernel<false><<<grid, 256, 0, s>>>(a, StridedSrc<kInF64>{d});
  else if (d.type == kInF16) dart_margin_kernel<false><<<grid, 256, 0, s>>>(a, StridedSrc<kInF16>{d});
  else throw Error("launch_dart_margin_inplace: element type " + std::to_string(d.type) + " is converted to float32 first (launch_convert_rows)");
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
