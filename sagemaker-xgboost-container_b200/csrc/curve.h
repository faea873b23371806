// curve.h -- the curve pass of `aucpr` (binary and one-vs-rest) and of multi-class `auc` (curve.cu; the scores come from
// misc.cu so they round like predict()).  DESIGN.md "AUC family" states the definitions.
#pragma once
#include "engine.h"

namespace b200 {

// scratch of one evaluation, kept on the Booster and grown on first use: the scores and row ids before and after the sort,
// each row's (positive, negative) mass and then its running sums, the sums at the tie-block ends, one double2 per tile of
// rows, the per-class (area, P, N) and the vector all-reduced across ranks
struct CurveScratch {
  DevBuf<float> key, key_sorted; DevBuf<int> iota, order, m; DevBuf<double2> cum, ends, tile;
  DevBuf<unsigned char> end_flag, tmp; DevBuf<double> part, cls, vec; DevBuf<unsigned> bad;
};

// misc.cu: key[i] = the score of row i (K == 0: the margin, through the sigmoid when logistic; K >= 2: the softmax
// probability of class c, as predict() computes it), -0.0 written as +0.0; iota[i] = i
void launch_curve_scores(const float* margin, int64_t n, int K, int c, int logistic, float* key, int* iota, cudaStream_t s);

// The per-rank vector of one metric on one matrix into sc->vec; returns its length (all-reduce it with a sum).
// pr = 0: ROC, K >= 2 only (binary auc stays in auc.cu); pr = 1: PR.  K == 0: binary, the labels are the positive
// share (checked to lie in [0, 1]); K >= 2: one-vs-rest over the softmax columns, positives (int)label == c.
int curve_metric_local(const float* margin, const float* label, const float* weight, int64_t n, int K, int logistic, int pr,
                       CurveScratch* sc, cudaStream_t s);
// The metric from the all-reduced vector: out[0] = value (nan when a class lacks positives or negatives), out[1] / out[2]
// = the global positive / negative weight (binary aucpr), out[3] = 1 when a label lies outside [0, 1] (binary aucpr)
void curve_metric_finish(int K, int pr, int world, CurveScratch* sc, double* out, cudaStream_t s);

}  // namespace b200
