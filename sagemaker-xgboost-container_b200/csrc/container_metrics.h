// container_metrics.h -- the device pass behind the container's own metrics (sagemaker_xgboost_container's custom_metrics:
// accuracy, f1, precision, recall, ..., and its scikit-learn mse / rmse / mae / r2).  DESIGN.md "Container metrics".
#pragma once
#include <vector>
#include "engine.h"

namespace b200 {

// label values a confusion matrix holds: labels 0 .. kContainerLabels - 1 (anything else leaves classification undecided)
constexpr int kContainerLabels = 64;
// the raw result: out[0] = bits of what was decided (kDecided*), out[1] = n, out[2] = P (predicted classes: 2 for one output
// per row, else the outputs), out[3] = kContainerLabels, out[4 .. 8) = float32 bits of sum (y - p)^2, sum |y - p|, sum y and
// sum (y - mean)^2 in numpy's pairwise order, out[8 ...] = the confusion counts [label][predicted class] (kContainerLabels x P)
constexpr int kContainerOutHead = 8;
constexpr int kContainerOutLen = kContainerOutHead + kContainerLabels * kContainerLabels;
enum : long long { kDecidedClass = 1, kDecidedReg = 2, kDecidedLabelSums = 4 };

// numpy's pairwise summation order for n float32 terms (numpy/_core/src/umath/loops_utils.h.src pairwise_sum): blocks of at
// most 128 terms summed with eight strided accumulators (fewer than 8 terms: in sequence), joined by the recursion that splits
// n at n/2 - (n/2 mod 8).  Nodes 0 .. leaves-1 are the blocks in order, node leaves + j is ops[j].x + ops[j].y, ops sorted by
// height (level_end[h] ends height h + 1); the root is the last node.  Depends only on n: built once per matrix.
struct PairwisePlan {
  int64_t n = -1; int leaves = 0;
  std::vector<int> level_end;
  DevBuf<int2> d_leaf;                     // (start, length) of each block
  DevBuf<int2> d_ops; DevBuf<int> d_level_end;
  void build(int64_t n, cudaStream_t s);
  int nodes() const { return leaves + (level_end.empty() ? 0 : level_end.back()); }
};

// per-matrix state: the plan and the label-only sums of r2 (sum y, sum (y - mean)^2), reset with the labels
struct ContainerSums {
  PairwisePlan plan;
  DevBuf<float> label_sums; bool labels_valid = false;
};

// per-call scratch kept on the Booster, grown on first use
struct ContainerScratch {
  DevBuf<float> terms;                     // [2 or 3][n] elementwise terms (regression metrics only)
  DevBuf<float> vals;                      // [2][nodes] block sums and the nodes above them
  DevBuf<long long> out;                   // kContainerOutLen
  void ensure(int64_t term_count, int64_t val_count);
};

struct ContainerArgs {
  const float* margin; const float* label; int64_t n;
  int K;                                   // outputs per row in the margins
  int objective, output_margin;
  int want_class, want_reg, want_r2;
};

// one pass over the rows, then the pairwise sums; leaves the raw result in sc->out (device)
void container_metrics_device(const ContainerArgs& a, ContainerSums* dm_sums, ContainerScratch* sc, cudaStream_t s);

}  // namespace b200
