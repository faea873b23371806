// adaptive.h -- reg:absoluteerror and reg:quantileerror: their gradient passes and the per-leaf quantile refresh of every tree ("adaptive tree",
// upstream src/objective/adaptive.{h,cc,cu} [UPSTREAM-RECALL]), an exact segmented radix select (adaptive.cu, DESIGN.md §3).
#pragma once
#include <functional>
#include "engine.h"

namespace b200 {

// Gradient pairs of reg:absoluteerror, same output contract as GradArgs: (sign(m - y) * w, w), rows the subsample draw
// rng_uniform(seed, 0x2000 + iter, r + row_offset) leaves out get (0, 0), max|g| and max h folded into absmax (may be nullptr);
// dense_g: g alone as float[n].  resid (may be nullptr): the round's residuals fl(y - m) of every row, sampled or not.
struct AbsErrGradArgs {
  const float* margin; const float* label; const float* weight;   // weight nullptr = 1
  float2* gpair; float* resid; unsigned* absmax;
  int64_t n, row_offset;
  float subsample; unsigned seed; unsigned long long iter; int dense_g;
};
void launch_abserr_gradient(const AbsErrGradArgs& a, cudaStream_t s);

// Gradient pairs of reg:quantileerror for Q targets from one label column: target j of row i gets, with d = fl(m[i][j] - y[i]),
// ((1 - alpha_j) w, w) when d >= 0 and (-alpha_j w, w) otherwise [UPSTREAM-RECALL: src/objective/quantile_obj.cu], all in
// float, into gpair[j * gp_stride + i]; margin is [n][Q] row-major, alpha Q floats on the device.  Rows outside the sample
// (the draw of AbsErrGradArgs, one per row for every target) get (0, 0); resid (may be nullptr) gets fl(y - m[i][j]) at
// [j * n + i] for every row.  dense_g (Q == 1 only): g alone as float[n].  absmax (may be nullptr): max|g| and max h of every
// target folded into [0] and [1], or with per_target those of target j into [2 j] and [2 j + 1] (2 Q entries), so that each
// target's trees can grow on a fixed-point grid of their own.
struct QuantileGradArgs {
  const float* margin; const float* label; const float* weight; const float* alpha;   // weight nullptr = 1
  float2* gpair; float* resid; unsigned* absmax;
  int64_t n, row_offset, gp_stride;
  float subsample; unsigned seed; unsigned long long iter; int dense_g, Q, per_target;
};
void launch_quantile_gradient(const QuantileGradArgs& a, cudaStream_t s);

// The quantile metric's sums: out[0] += sum_i sum_j fl(w_i * pinball_j(fl(y_i - m[i][j]))), out[1] += Q * sum_i w_i, in double
// (pinball_j(d) = fl(alpha_j d) for d >= 0, else fl(fl(alpha_j - 1) d)) [UPSTREAM-RECALL: src/metric/elementwise_metric.cu QuantileError]
void launch_quantile_metric(const float* margin, const float* label, const float* weight, const float* alpha, int Q, int64_t n, double* out,
                            cudaStream_t s);

// Selection state of one segment (a leaf).  mode 0: no rows; 1: the row of 0-based rank `target` in key order; 2: the first row
// in key order whose cumulative h_q reaches `target`.  d: upstream Quantile's interpolation weight, < 0 when the rank is clamped
// to an end (the value alone).  need_v1: the next larger key is not equal to the selected one and comes from the min pass.
struct SelectSeg { unsigned prefix; int mode; long long target; double d; int need_v1; int unused; };
static_assert(sizeof(SelectSeg) == 32, "SelectSeg layout");

constexpr int kSelectDigitBits = 4, kSelectBuckets = 1 << kSelectDigitBits, kSelectPasses = 32 / kSelectDigitBits;

// Device buffers of the selection, sized for up to `nseg` segments and `n` rows.
struct SelectScratch {
  DevBuf<unsigned long long> hist;        // [2][nseg][kSelectBuckets]: row counts, then h_q sums
  DevBuf<SelectSeg> st; DevBuf<unsigned> inv_min; DevBuf<float> q;
  DevBuf<int> seg;                        // per row: its segment, -1 = not selected from
  DevBuf<int> leaf_of_node, leaf_nid;     // training: dense leaf numbering of the tree's nodes
  DevBuf<float> resid;                    // training: the round's residuals, [targets][n]
  DevBuf<unsigned> absmax; DevBuf<float> scales;
  int nseg = 0;
  bool ensure(int64_t n, int nseg, int cap_nodes, int targets = 1);      // true when any buffer moved
};

// The selection proper.  values: per-row floats (-0.0 counts as +0.0, every NaN as one value above +inf); seg: per-row
// segment or -1; h (stride h_stride floats; nullptr = unweighted): the rows' weights, counted as h_q = rint(h * scales[1]), the fixed-point grid of the
// histograms.  alpha in [0, 1].  sum_i64 / max_u32 all-reduce the small per-pass arrays across ranks (no-ops on one GPU).
// On return sc->st and sc->q (per segment, NaN when empty) hold the result; with split_cond, the leaves
// leaf_nid[0 .. nseg) of a tree get fl(q * lr) unless empty.
struct SelectArgs {
  const float* values; const int* seg; const float* h; int h_stride; const float* scales;
  int64_t n; int nseg; double alpha;
  const int* leaf_nid; float* split_cond; float lr;
};
void segmented_select(const SelectArgs& a, SelectScratch* sc, const std::function<void(unsigned long long*, size_t)>& sum_i64,
                      const std::function<void(unsigned*, size_t)>& max_u32, cudaStream_t s);

// Training: each row's leaf (from node_of_row when the levels were routed, else from the root) as a dense leaf index into
// sc->seg, -1 for rows with h == 0 (gpair nullptr: none); the leaf numbering into sc->leaf_of_node / leaf_nid.
void launch_locate_leaves(const TreeArrays& t, const int* n_nodes, const uint8_t* bins_col, int64_t n, int has_missing,
                          const uint8_t* node_of_row, const float2* gpair, SelectScratch* sc, cudaStream_t s);

// sc->scales[1]: the fixed-point grid segmented_quantile counts `weights` on (the largest weight over all ranks, `global_n` rows).
// Training reads it when gradient-based sampling of weighted data weighs the refresh's rows by their instance weight.
void weight_grid(const float* weights, int64_t n, int64_t global_n, SelectScratch* sc, cudaStream_t s);

// The alpha-quantile of every segment over all ranks' rows (segs nullptr: one segment of every row; weights nullptr: unweighted;
// rows of weight 0 are left out), on the fixed-point grid of `global_n` rows.  out: nseg floats on the host, NaN when empty.
void segmented_quantile(const float* values, const int* segs, const float* weights, int64_t n, int64_t global_n, int nseg, double alpha,
                        float* out, SelectScratch* sc, cudaStream_t s);

}  // namespace b200
