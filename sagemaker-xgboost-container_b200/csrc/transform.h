// transform.h -- predict()'s margin -> prediction transform (upstream PredTransform), shared by predict() (misc.cu) and the
// container metrics (container_metrics.cu), which must read predict()'s values bit for bit.  expf's inlined code contains a
// multiply-add, so every file that includes this header is compiled with the default --fmad=true.
#pragma once
#include "engine.h"

namespace b200 {

__device__ __forceinline__ float sigmoidf_xgb(float x) {
  const float kEps = 1e-16f;
  x = fminf(-x, 88.7f);
  float denom = expf(x) + 1.0f + kEps;
  return 1.0f / denom;
}
// softmax of the margins p[0, K): returns the sum of expf(p[k] - wmax) over k, with wmax the largest margin; class k's
// probability is expf(p[k] - wmax) / sum (predict() and the multi-class auc / aucpr scores)
__device__ __forceinline__ float softmax_sum(const float* p, int K, float* wmax_out) {
  float wmax = p[0];
  for (int k = 1; k < K; ++k) if (p[k] > wmax) wmax = p[k];
  float wsum = 0.f;
  for (int k = 0; k < K; ++k) wsum += expf(p[k] - wmax);
  *wmax_out = wmax;
  return wsum;
}
// multi:softmax's prediction: the first largest margin (a NaN margin is never taken after p[0])
__device__ __forceinline__ int softmax_class(const float* p, int K) {
  float wmax = p[0]; int arg = 0;
  for (int k = 1; k < K; ++k) if (p[k] > wmax) { wmax = p[k]; arg = k; }
  return arg;
}
// the prediction of an objective with one output per row
__device__ __forceinline__ float transform_one(float m, int objective) {
  if (objective == kBinaryLogistic || objective == kRegLogistic) return sigmoidf_xgb(m);
  if (objective == kPoisson || objective == kGamma || objective == kTweedie || objective == kAft || objective == kCox) return expf(m);
  if (objective == kHinge) return m > 0.0f ? 1.0f : 0.0f;
  return m;
}

}  // namespace b200
