// multi_target.h -- multi-target regression (DESIGN.md "Multi-target regression"): T label columns, one tree per target per
// round.  The gradient and metric passes over the n x T label elements (multi_target.cu).
#pragma once
#include "engine.h"

namespace b200 {

// the objectives that train on a label of T > 1 columns: the RegLossObj family, reg:pseudohubererror and reg:absoluteerror
inline bool objective_is_multi_target(int o) {
  return o == kSquaredError || o == kSquaredLogError || o == kPseudoHuber || o == kRegLogistic || o == kBinaryLogistic || o == kLogitRaw ||
         o == kAbsoluteError;
}

// Gradient pairs of T targets: target j of row i is gradient_kernel's pair of one element, computed from y = label[i][j],
// m = margin[i][j] (label and margin [n][T] row-major, margin nullptr = 0) and the row's weight w_i (nullptr = 1; times
// scale_pos_weight when y == 1 under the RegLossObj family), into gpair[j * gp_stride + i].  reg:absoluteerror gets
// (sign(m - y) w, w) and its residuals fl(y - m) into resid[j * n + i] (resid may be nullptr).  Rows outside the sample draw
// (one per row, shared by the targets) get (0, 0).  absmax (may be nullptr): each target's max|g| and max h into [2 j] and
// [2 j + 1], or with per_target == 0 all of them into [0] and [1].  err: gradient_kernel's label-range codes.
struct MultiGradArgs {
  const float* margin; const float* label; const float* weight;
  float2* gpair; float* resid; unsigned* absmax; int* err;
  int64_t n, row_offset, gp_stride;
  int T, objective, per_target;
  float scale_pos_weight, subsample, aux;
  unsigned seed; unsigned long long iter;
};
void launch_multi_target_gradient(const MultiGradArgs& a, cudaStream_t s);

// An element-wise metric over the n x T elements: out[0] += sum_i sum_j fl(loss(y_ij, p_ij) * w_i), out[1] += T * sum_i w_i, in
// double; p_ij is the margin through the objective's transform (misc.h MetricArgs: metric, is_logistic, transform, threshold, aux).
struct MultiMetricArgs {
  const float* margin; const float* label; const float* weight; double* out;
  int64_t n; int T, metric, is_logistic, transform; float threshold, aux;
};
void launch_multi_target_metric(const MultiMetricArgs& a, cudaStream_t s);

// out[i] = label[i * T + j]: label column j, contiguous (the per-target median of the intercept)
void launch_label_column(const float* label, int64_t n, int T, int j, float* out, cudaStream_t s);

}  // namespace b200
