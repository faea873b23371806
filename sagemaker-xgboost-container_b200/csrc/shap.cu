// shap.cu -- per-feature prediction contributions (Booster.predict(pred_contribs=True), SURVEY.md section 8a row A12; the
// container's integration test calls it at test/integration/local/test_abalone.py:65).
// Algorithm: path-dependent Tree SHAP (Lundberg et al.) in the formulation of upstream xgboost's src/predictor/cpu_treeshap.cc
// [UPSTREAM-RECALL v3.0.5]: a depth-first walk that carries the set of unique features on the path with, per feature, the
// fraction of "zero" (feature unknown: both children, weighted by cover = sum_hess) and "one" (feature known: the row's child)
// paths and the permutation weights; a split on a feature already on the path first unwinds that feature.
// One thread per row, trees in model order, float arithmetic like upstream.  The recursion is an explicit stack; a node's
// path copy lives at parent + unique_depth + 1 in a triangular per-thread array exactly like upstream's unique_path_data.
// Low-volume serving call, not a training hot path: no shared-memory staging of the model.
#include <cmath>
#include "engine.h"
#include "misc.h"

namespace b200 {

struct PathElement { int feature; float zero_fraction, one_fraction, pweight; };
struct ShapFrame { int node, depth, parent_off; float zero_fraction, one_fraction; int feature; };

__device__ __forceinline__ void extend_path(PathElement* p, int depth, float zf, float of, int feature) {
  p[depth].feature = feature; p[depth].zero_fraction = zf; p[depth].one_fraction = of; p[depth].pweight = depth == 0 ? 1.0f : 0.0f;
  for (int i = depth - 1; i >= 0; --i) {
    p[i + 1].pweight += of * p[i].pweight * (float)(i + 1) / (float)(depth + 1);
    p[i].pweight = zf * p[i].pweight * (float)(depth - i) / (float)(depth + 1);
  }
}

__device__ __forceinline__ void unwind_path(PathElement* p, int depth, int index) {
  const float of = p[index].one_fraction, zf = p[index].zero_fraction;
  float next_one = p[depth].pweight;
  for (int i = depth - 1; i >= 0; --i) {
    if (of != 0.0f) {
      const float tmp = p[i].pweight;
      p[i].pweight = next_one * (float)(depth + 1) / ((float)(i + 1) * of);
      next_one = tmp - p[i].pweight * zf * (float)(depth - i) / (float)(depth + 1);
    } else {
      p[i].pweight = (p[i].pweight * (float)(depth + 1)) / (zf * (float)(depth - i));
    }
  }
  for (int i = index; i < depth; ++i) { p[i].feature = p[i + 1].feature; p[i].zero_fraction = p[i + 1].zero_fraction; p[i].one_fraction = p[i + 1].one_fraction; }
}

__device__ __forceinline__ float unwound_path_sum(const PathElement* p, int depth, int index) {
  const float of = p[index].one_fraction, zf = p[index].zero_fraction;
  float next_one = p[depth].pweight, total = 0.0f;
  for (int i = depth - 1; i >= 0; --i) {
    if (of != 0.0f) {
      const float tmp = next_one * (float)(depth + 1) / ((float)(i + 1) * of);
      total += tmp;
      next_one = p[i].pweight - tmp * zf * ((float)(depth - i) / (float)(depth + 1));
    } else if (zf != 0.0f) {
      total += (p[i].pweight / zf) / ((float)(depth - i) / (float)(depth + 1));
    }
  }
  return total;
}

template <int MAXD>          // MAXD = deepest tree + 2
__global__ void __launch_bounds__(128) shap_kernel(ShapArgs a) {
  constexpr int kPath = MAXD * (MAXD + 1) / 2;
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n) return;
  PathElement path[kPath];
  ShapFrame stack[MAXD + 2];
  const float* x = a.X + r * a.F;
  const int cols = a.F + 1;
  for (int t = a.tree_begin; t < a.tree_end; ++t) {
    const ShapNode* nodes = a.nodes + a.tree_offset[t - a.tree_begin];
    float* phi = a.out + (r * a.K + a.tree_info[t - a.tree_begin]) * cols;
    const float tw = a.tree_weight ? a.tree_weight[t - a.tree_begin] : 1.0f;     // booster=dart: the tree's weight
    int sp = 0;
    stack[sp++] = ShapFrame{0, 0, 0, 1.0f, 1.0f, -1};
    while (sp > 0) {
      const ShapFrame fr = stack[--sp];
      const PathElement* parent = path + fr.parent_off;
      int depth = fr.depth;
      const int my_off = fr.parent_off + depth + 1;
      PathElement* up = path + my_off;
      for (int i = 0; i <= depth; ++i) up[i] = parent[i];
      extend_path(up, depth, fr.zero_fraction, fr.one_fraction, fr.feature);
      const ShapNode nd = nodes[fr.node];
      if (nd.left < 0) {
        for (int i = 1; i <= depth; ++i) {
          const float w = unwound_path_sum(up, depth, i);
          if (a.tree_weight) phi[up[i].feature] += (w * (up[i].one_fraction - up[i].zero_fraction) * nd.cond) * tw;
          else phi[up[i].feature] += w * (up[i].one_fraction - up[i].zero_fraction) * nd.cond;
        }
      } else {
        const int split = (int)(nd.fidx_dl & 0x7fffffffu);
        const float fv = split < a.F ? x[split] : nanf("");
        const bool go_left = isnan(fv) ? (nd.fidx_dl >> 31) != 0 : fv < nd.cond;
        const int hot = go_left ? nd.left : nd.right, cold = go_left ? nd.right : nd.left;
        const float w = nd.sum_hess;
        const float hot_zero = nodes[hot].sum_hess / w, cold_zero = nodes[cold].sum_hess / w;
        float incoming_zero = 1.0f, incoming_one = 1.0f;
        int pi = 0;
        for (; pi <= depth; ++pi) if (up[pi].feature == split) break;
        if (pi != depth + 1) {
          incoming_zero = up[pi].zero_fraction; incoming_one = up[pi].one_fraction;
          unwind_path(up, depth, pi);
          depth -= 1;
        }
        // the hot child is walked first (popped first), like upstream's recursion order
        stack[sp++] = ShapFrame{cold, depth + 1, my_off, cold_zero * incoming_zero, 0.0f, split};
        stack[sp++] = ShapFrame{hot, depth + 1, my_off, hot_zero * incoming_zero, incoming_one, split};
      }
    }
    if (a.tree_weight) phi[a.F] += nodes[0].mean * tw;
    else phi[a.F] += nodes[0].mean;     // expected value of the tree (cover-weighted mean of its leaves)
  }
}

__global__ void shap_bias_kernel(float* out, const float* base_margin_rows, float base_margin, int64_t n, int K, int cols) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n * K) out[i * cols + cols - 1] += base_margin_rows ? base_margin_rows[i] : base_margin;
}

void launch_shap(const ShapArgs& a, int max_depth, cudaStream_t s) {
  if (a.n == 0) return;
  const unsigned grid = (unsigned)((a.n + 127) / 128);
  const int maxd = max_depth + 2;
  if (maxd <= 8) shap_kernel<8><<<grid, 128, 0, s>>>(a);
  else if (maxd <= 12) shap_kernel<12><<<grid, 128, 0, s>>>(a);
  else if (maxd <= 18) shap_kernel<18><<<grid, 128, 0, s>>>(a);
  else if (maxd <= 34) shap_kernel<34><<<grid, 128, 0, s>>>(a);
  else throw Error("pred_contribs: trees deeper than 32 levels are not supported");
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
  shap_bias_kernel<<<(unsigned)((a.n * a.K + 255) / 256), 256, 0, s>>>(a.out, a.base_margin_rows, a.base_margin, a.n, a.K, a.F + 1);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
