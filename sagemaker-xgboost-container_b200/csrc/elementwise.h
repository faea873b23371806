// elementwise.h -- the per-element gradient of the single-output regression objectives and the per-element loss of the
// element-wise metrics, shared by gradient_kernel / metric_kernel (misc.cu) and their multi-target siblings (multi_target.cu),
// so that target j of a multi-target model computes what a single-target model trained on label column j computes, bit for
// bit.  Both files keep the default --fmad=true (see transform.h).
#pragma once
#include "engine.h"
#include "misc.h"
#include "transform.h"

namespace b200 {

// the RegLossObj family (reg:squarederror, reg:logistic, binary:logistic, binary:logitraw, reg:squaredlogerror,
// reg:pseudohubererror): scale_pos_weight multiplies the weight of a row whose label is 1
__device__ __forceinline__ bool objective_is_reg_loss(int o) { return o <= kLogitRaw || o == kSquaredLogError || o == kPseudoHuber; }

// (g, h) of one element before the weight: upstream src/objective/regression_loss.h (RegLossObj family), regression_obj.cu
// (Poisson / Gamma / Tweedie), hinge.cu.  *err gets gradient_kernel's label-range codes (misc.h GradArgs).
__device__ __forceinline__ void elementwise_gradient(int objective, float y, float p, float aux, int* err, float* g_out, float* h_out) {
  float g, h;
  switch (objective) {
    case kSquaredError: g = p - y; h = 1.0f; break;
    case kSquaredLogError: {
      if (!(y > -1.0f)) *err = 3;
      p = fmaxf(p, -1.0f + 1e-6f);
      g = (log1pf(p) - log1pf(y)) / (p + 1.0f);
      h = fmaxf((-log1pf(p) + log1pf(y) + 1.0f) / ((p + 1.0f) * (p + 1.0f)), 1e-6f);
      break; }
    case kPseudoHuber: {
      const float z = p - y, s2 = aux * aux, scale_sqrt = sqrtf(1.0f + z * z / s2);
      g = z / scale_sqrt; h = s2 / ((s2 + z * z) * scale_sqrt);
      break; }
    case kPoisson: {
      if (y < 0.0f) *err = 4;
      g = expf(p) - y; h = expf(p + aux);
      break; }
    case kGamma: {
      if (!(y > 0.0f)) *err = 5;
      const float ep = expf(p);
      g = 1.0f - y / ep; h = y / ep;
      break; }
    case kTweedie: {
      if (y < 0.0f) *err = 6;
      const float rho = aux, e1 = expf((1.0f - rho) * p), e2 = expf((2.0f - rho) * p);
      g = -y * e1 + e2; h = -y * (1.0f - rho) * e1 + (2.0f - rho) * e2;
      break; }
    case kHinge: {
      const float yy = y * 2.0f - 1.0f;
      if (p * yy < 1.0f) { g = -yy; h = 1.0f; } else { g = 0.0f; h = 1.17549435e-38f; }      // upstream: numeric_limits<float>::min()
      break; }
    default: {
      if (y < 0.0f || y > 1.0f) *err = 1;
      p = sigmoidf_xgb(p); g = p - y; h = fmaxf(p * (1.0f - p), 1e-16f);
      break; }
  }
  *g_out = g; *h_out = h;
}

// the loss of one element of an element-wise metric at prediction p (the transform already applied); upstream
// src/metric/elementwise_metric.cu
__device__ __forceinline__ float elementwise_loss(int metric, float y, float p, float threshold, float aux) {
  float loss = 0.f;
  switch (metric) {
    case kMetricRmsle: { float d = log1pf(y) - log1pf(p); loss = d * d; break; }
    case kMetricMape: loss = fabsf((y - p) / y); break;
    case kMetricMphe: { const float z = (y - p) / aux; loss = aux * aux * (sqrtf(1.0f + z * z) - 1.0f); break; }
    case kMetricPoissonNll: { const float py = fmaxf(p, 1e-16f); loss = lgammaf(y + 1.0f) + py - logf(py) * y; break; }
    case kMetricGammaNll: { const float py = fmaxf(p, 1e-6f); loss = y / py + logf(py); break; }       // psi = 1: -((y * theta - b) / a + c), theta = -1 / py, b = -log(-theta)
    case kMetricGammaDeviance: { const float py = p + 1e-6f, yy = y + 1e-6f; loss = logf(py / yy) + yy / py - 1.0f; break; }      // x 2 on the host
    case kMetricTweedieNll: { const float rho = aux, lp = logf(p); loss = -y * expf((1.0f - rho) * lp) / (1.0f - rho) + expf((2.0f - rho) * lp) / (2.0f - rho); break; }
    case kMetricRmse: { float d = p - y; loss = d * d; break; }
    case kMetricMae: loss = fabsf(p - y); break;
    case kMetricLogloss: {
      const float eps = 1e-16f;
      float pneg = 1.0f - p;
      if (p < eps) loss = -y * logf(eps) - (1.0f - y) * logf(1.0f - eps);
      else if (pneg < eps) loss = -y * logf(1.0f - eps) - (1.0f - y) * logf(eps);
      else loss = -y * logf(p) - (1.0f - y) * logf(pneg);
      break; }
    case kMetricError: loss = (p > threshold) ? (1.0f - y) : y; break;
    default: break;
  }
  return loss;
}

// the metric's view of a margin: the objective's transform (is_logistic: binary:logitraw under logloss / error)
__device__ __forceinline__ float metric_prediction(float m, int is_logistic, int transform) {
  if (is_logistic || transform == kTransformSigmoid) return sigmoidf_xgb(m);
  if (transform == kTransformExp) return expf(m);
  if (transform == kTransformHinge) return m > 0.0f ? 1.0f : 0.0f;
  return m;
}

}  // namespace b200
