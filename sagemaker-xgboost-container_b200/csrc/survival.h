// survival.h -- survival:aft and survival:cox objectives and their metrics (survival.cu)
#pragma once
#include "engine.h"

namespace b200 {

// aft_loss_distribution (upstream ProbabilityDistributionType)
enum AftDist : int { kAftNormal = 0, kAftLogistic = 1, kAftExtreme = 2 };

// Gradient pairs of a survival objective.  Same output contract as GradArgs: gpair[r] = (g * w, h * w), rows the subsample
// draw rng_uniform(seed, 0x2000 + iter, r + row_offset) leaves out get (0, 0), max|g| and max h folded into absmax (may be nullptr).
struct SurvivalGradArgs {
  const float* margin;                  // n rows
  const float* label;                   // survival:cox: event time y > 0, censored at |y| when y <= 0
  const float* lower; const float* upper;   // survival:aft: interval bounds (upper may be +inf)
  const float* weight;                  // nullptr = 1
  float2* gpair; unsigned* absmax;
  int64_t n, row_offset;
  float subsample; unsigned seed; unsigned long long iter;
  int dist; float sigma;                // survival:aft: distribution and scale
};

// survival:cox: the rows in stable ascending |label| order, the sorted position of each position's tie-group head, and the
// event flag in sorted order.  Built once per label set (cox_sort) and cached on the DMatrix.
struct CoxOrder {
  DevBuf<int> order, head; DevBuf<unsigned char> event;
  int64_t n = 0; bool valid = false;
};

// per-round scratch of the Cox gradient and metric: exp(margin) in sorted order, its suffix sums, the (R, S) scan, tile sums
struct CoxScratch {
  DevBuf<double> e, suffix; DevBuf<double2> rs, tiles; DevBuf<unsigned char> tmp;
  void ensure(int64_t n);
};

void launch_aft_gradient(const SurvivalGradArgs& a, cudaStream_t s);
void cox_sort(const float* label, int64_t n, CoxOrder* o, CoxScratch* sc, cudaStream_t s);
void launch_cox_gradient(const SurvivalGradArgs& a, const CoxOrder& o, CoxScratch* sc, cudaStream_t s);

// metrics on raw margins.  aft: out[0] += sum(w * loss), out[1] += sum(w); metric 0 = aft-nloglik, 1 = interval-regression-accuracy.
// cox: out[0] = -sum over events of (m_i - ln D_i), out[1] = the number of events (written, not added; deterministic)
void launch_aft_metric(const float* margin, const float* lower, const float* upper, const float* weight, int64_t n, int dist, float sigma,
                       int metric, double* out, cudaStream_t s);
void cox_nloglik(const float* margin, int64_t n, const CoxOrder& o, CoxScratch* sc, double* out, cudaStream_t s);

}  // namespace b200
