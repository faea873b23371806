// split_math.h -- the node weight and gain arithmetic of the tree builder (tree.cu), shared with the tree refresh (refresh.cu)
// so that a refreshed node's statistics are computed by the very functions that grew it.
// The float/double mix follows upstream src/tree/param.h + split_evaluator.h.
#pragma once
#include "tree.h"

namespace b200 {

__device__ __forceinline__ double threshold_l1(double w, double alpha) {
  if (w > +alpha) return w - alpha;
  if (w < -alpha) return w + alpha;
  return 0.0;
}
__device__ __forceinline__ float calc_weight(const TrainParamDev& p, double G, double H) {
  if (H < p.min_child_weight || H <= 0.0) return 0.0f;
  double dw = -threshold_l1(G, p.alpha) / (H + p.lambda);
  if (p.max_delta_step != 0.0f && fabs(dw) > p.max_delta_step) dw = copysign((double)p.max_delta_step, dw);
  return (float)dw;
}
// -(2 g w + (h + lambda) w^2) in float with every product rounded before the add, as upstream's CPU code evaluates it: a fused
// multiply-add would change the last bits of loss_chg, and at near-ties which split wins
__device__ __forceinline__ float gain_at_weight_f(float g, float h, float lambda, float w) {
  return -__fadd_rn(__fmul_rn(__fmul_rn(2.0f, g), w), __fmul_rn(__fmul_rn(__fadd_rn(h, lambda), w), w));
}
__device__ __forceinline__ float calc_gain_given_weight(const TrainParamDev& p, double G, double H, float w) {
  if (H <= 0.0) return 0.0f;
  if (p.max_delta_step == 0.0f) { double t = threshold_l1(G, p.alpha); return (float)(t * t / (H + p.lambda)); }
  return gain_at_weight_f((float)G, (float)H, p.lambda, w);
}
__device__ __forceinline__ float calc_gain(const TrainParamDev& p, double G, double H) {
  return calc_gain_given_weight(p, G, H, calc_weight(p, G, H));
}
__device__ __forceinline__ float calc_split_gain(const TrainParamDev& p, double GL, double HL, double GR, double HR) {
  float wl = calc_weight(p, GL, HL), wr = calc_weight(p, GR, HR);
  return calc_gain_given_weight(p, GL, HL, wl) + calc_gain_given_weight(p, GR, HR, wr);
}

}  // namespace b200
