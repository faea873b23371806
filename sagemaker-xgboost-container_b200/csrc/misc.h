// misc.h -- argument blocks and launchers for misc.cu / quantile.cu
#pragma once
#include "engine.h"
#include "inplace.h"
#include "predict_plan.h"

namespace b200 {

struct GradArgs {
  const float* margin;      // n x K row-major, nullptr = all zero (base-score stump)
  const float* label; const float* weight;
  float2* gpair;            // [K][gp_stride]
  int64_t gp_stride;        // rows reserved per class (>= n, multiple of 64: keeps class blocks 16 B aligned for the TMA bulk copies)
  int dense_g;              // constant-hessian objectives (K == 1, h == 1 for every row): gpair holds float g[gp_stride] instead of the
                            // pairs; max h (1.0f) is folded into absmax as for the pairs
  unsigned* absmax;         // max|g|, max h as float bits (atomicMax), may be nullptr
  int* err;                 // 1 = logistic label range, 2 = multiclass label range, 3 = squaredlogerror label <= -1, 4 = poisson label < 0,
                            // 5 = gamma label <= 0, 6 = tweedie label < 0
  int64_t n, row_offset;    // row_offset: global index of local row 0 (multi-GPU subsampling stream)
  int K, objective;
  float scale_pos_weight, subsample;
  unsigned seed; unsigned long long iter;
  float aux;                // objective parameter: huber_slope / tweedie_variance_power / the Poisson max_delta_step
};

struct DevNode { float cond; int left; int right; unsigned fidx_dl; };   // 16 B, leaf: left == -1, cond = leaf value

struct PredictArgs {
  const float* X; int64_t n; int F;
  const DevNode* nodes; const int64_t* tree_offset; const int* tree_info;
  int tree_begin, tree_end, K;
  float* margin;            // n x K, pre-initialised with the base margin; may be nullptr
  int* leaf;                // n x (tree_end - tree_begin); may be nullptr
  const int64_t* h_tree_offset;   // host copy of tree_offset (plans the shared-memory tree chunks); nullptr = thread-per-row kernel
  int has_nan;              // the matrix contains missing values
  int children_adjacent;    // right child == left child + 1 in every tree (true for every tree this engine trains)
  int model_F;              // features of the model: a matrix with F < model_F reads the features it lacks as missing
};

enum Metric : int { kMetricRmse = 0, kMetricMae = 1, kMetricLogloss = 2, kMetricError = 3, kMetricMerror = 4, kMetricMlogloss = 5,
                    kMetricAuc = 6, kMetricMse = 7, kMetricRmsle = 8, kMetricMape = 9, kMetricMphe = 10, kMetricPoissonNll = 11,
                    kMetricGammaNll = 12, kMetricGammaDeviance = 13, kMetricTweedieNll = 14 };

struct MetricArgs {
  const float* margin; const float* label; const float* weight; double* out;
  int64_t n; int K, metric, is_logistic; float threshold;
  int transform;            // engine.h Transform applied to the margin first (is_logistic == 1 is kTransformSigmoid)
  float aux;                // huber slope (mphe) / variance power (tweedie-nloglik)
};

// prediction contributions (shap.cu): the model subset [tree_begin, tree_end) repacked with cover and mean value per node
struct ShapNode { float cond; int left; int right; unsigned fidx_dl; float sum_hess; float mean; };   // leaf: left == -1, cond = leaf value
struct ShapArgs {
  const float* X; int64_t n; int F;
  const ShapNode* nodes; const int64_t* tree_offset; const int* tree_info;     // offsets / classes indexed from tree_begin
  int tree_begin, tree_end, K;
  float* out;                      // [n][K][F + 1], zero-initialised by the caller
  const float* base_margin_rows;   // [n][K] user base margins, or nullptr -> base_margin
  float base_margin;
  const float* tree_weight;        // per tree from tree_begin: its contributions are multiplied by it (booster=dart); nullptr = 1
};
void launch_shap(const ShapArgs& a, int max_depth, cudaStream_t s);

// booster=dart (dart.cu): the leaf values of the listed trees on each row, weighted, into the margins [n][K]
struct DartArgs {
  const float* X; int64_t n; int F;
  const DevNode* nodes; const int64_t* tree_offset; const int* tree_info;   // the device model, indexed by tree id
  const int* trees; int ntrees; int K;          // the listed tree ids, in the order they are added
  const float* coef_full;                       // per listed tree: m_full += fl(coef_full * leaf)
  const float* coef_drop;                       // per listed tree: m_drop -= fl(coef_drop * leaf); unused without m_drop
  float* m_full;
  float* m_drop;                                // nullptr = no dropped margin; else written as m_full minus the dropped trees
};
void launch_dart_margin(const DartArgs& a, cudaStream_t s);
// the same pass (no dropped margin) reading the in-place input d instead of a.X (d: float32, float64, float16 or CSR)
void launch_dart_margin_inplace(const DartArgs& a, const InputDesc& d, cudaStream_t s);

// num_parallel_tree > 1 with subsample < 1: one tree's row sample of the round's unsampled gradients (misc.cu)
struct SampleArgs {
  const float2* src;        // [K][gp_stride] the round's gradients, every row
  float2* dst;              // [K][gp_stride] the tree's copy: unsampled rows get (0, 0)
  unsigned* absmax;         // max|g|, max h of dst as float bits (atomicMax)
  int64_t gp_stride, n, row_offset;
  int K; float subsample; unsigned seed; unsigned long long stream;
};

void launch_gradient(const GradArgs& a, cudaStream_t s);
void launch_sample_gpair(const SampleArgs& a, cudaStream_t s);
void launch_sum_gpair(const float2* gp, int64_t n, double* out, cudaStream_t s);
void launch_bin(const float* X, int64_t n, int F, int ngroups, int tw, const int* cut_ptrs, const float* cut_vals, uint8_t* bins, uint8_t* bins_tail, cudaStream_t s);
void launch_transpose_bins(const uint8_t* bins, const uint8_t* bins_tail, int64_t n, int F, int ngroups, int tw, uint8_t* bins_col, cudaStream_t s);
void launch_pad_rows(const uint8_t* src, const uint8_t* tail, int tw, int64_t n, int src_stride, uint8_t* dst, int dst_stride, cudaStream_t s);
void launch_count_nan(const float* X, int64_t count, float missing, int use_missing, unsigned long long* out, cudaStream_t s);
void launch_replace_missing(float* X, int64_t count, float missing, cudaStream_t s);
PredictPlan plan_for(const PredictArgs& a);             // what launch_predict(a) runs
void launch_predict(const PredictArgs& a, cudaStream_t s);
// launch_predict's plan on the in-place input d (inplace.h; float32, float64, float16 or CSR) instead of a.X: margins only,
// always the NaN-aware variant (no pass over the input decides has_nan)
void launch_predict_inplace(const PredictArgs& a, const InputDesc& d, cudaStream_t s);
// rows [r0, r0 + rows) of d converted to float32 into out (rows x d.F, row-major, NaN = missing): the element types the
// predictor does not read itself, a bounded tile at a time
void launch_convert_rows(const InputDesc& d, int64_t r0, int64_t rows, float* out, cudaStream_t s);
// Prediction from the bins (predict_bins.cu).  Each value stands at the lower edge of its bin (min_vals[f] for bin 0, else
// cut_vals[ptr + b - 1]), so `x < cond` becomes `b < t` with t the number of the feature's lower edges below cond.
// launch_bin_thresholds copies nodes[0, count) to out with each split's cond replaced by t (as int bits); a split on a feature
// f >= F reads feature 0 with t fixed to its default direction (0: right, 512: left).
void launch_bin_thresholds(const DevNode* nodes, size_t count, const int* cut_ptrs, const float* cut_vals, const float* min_vals, int F,
                           DevNode* out, cudaStream_t s);
PredictPlan plan_for_bins(const PredictArgs& a, const BinnedMatrix& m);   // what launch_predict_bins(a, m) runs
// launch_predict on m's bins: a.nodes are launch_bin_thresholds' nodes; a.X and a.has_nan are not read (m.has_missing is)
void launch_predict_bins(const PredictArgs& a, const BinnedMatrix& m, cudaStream_t s);
void launch_transform(float* m, int64_t n, int K, int objective, float* out_class, cudaStream_t s);
void launch_fill(float* p, int64_t n, float v, cudaStream_t s);
void launch_metric(const MetricArgs& a, cudaStream_t s);
// auc.cu (experimental): out[0] += unnormalised ROC area, out[1] = positive weight, out[2] = negative weight
void compute_auc_device(const float* margin, const float* label, const float* weight, int64_t n, int is_logistic, double* out, cudaStream_t s);

// quantile.cu: exact weighted-quantile cuts per feature (same definition as oracle/gbt_oracle.c cuts_from_distinct).
// X: device, row-major n x F. Returns host vectors.
struct HostCuts { std::vector<int> ptrs; std::vector<float> vals; std::vector<float> mins; };
void compute_cuts_device(const float* dX, int64_t n, int F, const float* dweights, int max_bin, bool has_missing,
                         HostCuts* out, cudaStream_t s);
// Distinct-value summary of one rank (for merging cuts across ranks): per feature the sorted distinct values and
// their weights (summed in double, in an order fixed by the input), exact when a feature has <= cap distinct values, else
// a cap-point weighted-quantile summary.  A column that holds +inf and missing values keeps +inf as a value.
struct FeatureSummary { std::vector<float> vals; std::vector<double> weights; };
void compute_summaries_device(const float* dX, int64_t n, int F, const float* dweights, int cap,
                              std::vector<FeatureSummary>* out, cudaStream_t s);
void cuts_from_summaries(const std::vector<FeatureSummary>& sums, int max_bin, bool has_missing, HostCuts* out);
// Multi-rank cuts: every rank summarises its shard with at most kRankSummaryCap points per feature (exact while the shard
// has no more distinct values), and merge_summaries joins the summaries of all ranks, taken in rank order: a stable sort by
// value, equal values adding their weights.  compute_rank_cuts_device runs that recipe on one GPU over the row ranges
// [row_bounds[r], row_bounds[r + 1]) of one matrix, as if each range were a rank's shard.
constexpr int kRankSummaryCap = 2048;
void merge_summaries(const std::vector<std::vector<FeatureSummary>>& per_rank, int F, std::vector<FeatureSummary>* merged);
void compute_rank_cuts_device(const float* dX, int F, const float* dweights, const int64_t* row_bounds, int nranges, int max_bin,
                              bool has_missing, HostCuts* out, cudaStream_t s);

// tree_method=approx (DESIGN.md "Approx"): what a matrix keeps to re-sketch its cuts before every tree on the device.  Only the
// A features with more distinct values than bins are kept (the cuts of the others do not depend on the weights): each one's
// non-missing rows in value order and the runs of equal values in that order.
struct ApproxSketch {
  bool valid = false;
  int64_t n = 0; int F = 0, nb = 0, A = 0; int64_t nruns = 0;
  DevBuf<int> order;                 // kept feature a: rows [elem_off[a], elem_off[a + 1]) in value order
  DevBuf<int64_t> elem_off;          // [A + 1]
  DevBuf<int> run_start;             // [nruns]: a run's first entry, relative to its feature's elem_off
  DevBuf<int64_t> run_off;           // [A + 1]: feature a's runs
  DevBuf<int> feat;                  // [A]: the feature id of kept feature a
  DevBuf<double> run_w;              // [nruns]: per tree, each run's weight, then its inclusive cumulative weight
  DevBuf<float> stage_vals;          // [F][256]: each feature's cuts before they are packed (the others' fixed cuts from the start)
  DevBuf<int> stage_cnt;             // [F]
};
// out[r] = gp[r].y for r < n: one class's hessian as row weights (the multi-rank re-sketch)
void launch_hessian_column(const float2* gp, int64_t n, float* out, cudaStream_t s);
// Built once per matrix (host-synchronising, like the one-time cuts): nb bins per feature, `cuts` the matrix's own cuts.
void approx_sketch_build(const float* dX, int64_t n, int F, int nb, const HostCuts& cuts, ApproxSketch* sk, cudaStream_t s);
// The cuts of one tree with weights gp[r].y (the tree's hessian) into cut_ptrs ([F + 1]) and cut_vals ([F][256] capacity),
// in launches only.  The min values do not change: they depend on each feature's first value alone.
void approx_sketch_cuts(const float* dX, const ApproxSketch& sk, const float2* gp, int* cut_ptrs, float* cut_vals, cudaStream_t s);

}  // namespace b200
