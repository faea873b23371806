// rank.h -- rank:pairwise, rank:ndcg and rank:map over query groups (LambdaRank gradients over the topk pairs) and the
// ndcg / map metrics (rank.cu).  DESIGN.md "Learning to rank" states the formulas.
#pragma once
#include <vector>
#include "engine.h"

namespace b200 {

// A DMatrix's query groups on the device: the group pointer (one group of every row when the matrix has none), the group
// of each row, and the labels sorted descending within each group.  Built on first use, reset with the labels, groups or weights.
struct RankGroups {
  DevBuf<int> ptr, row_group; DevBuf<float> ideal; DevBuf<int> ideal_order;   // ideal_order: the rows in that label order
  int64_t n = 0, G = 0; bool valid = false;
};

// scratch of one gradient or metric call: the margins, labels and row ids in sorted order, the MAP prefix sums (hits, sum of
// 1 / (r + 1) over the hits), the per-document pair sums (g, h, |lambda|) and one double per group
struct RankScratch {
  DevBuf<float> key, key_sorted, y_sorted; DevBuf<int> iota, order; DevBuf<double2> hq; DevBuf<double> acc, group; DevBuf<unsigned char> tmp;
  DevBuf<int> pos; DevBuf<unsigned long long> fix;      // mean pairs: each row's position in the margin order, fixed-point sums
};

// Same output contract as GradArgs: gpair[r] = (g, h) of row r, rows the subsample draw rng_uniform(seed, 0x2000 + iter,
// r + row_offset) leaves out get (0, 0), max|g| and max h folded into absmax (may be nullptr).
struct RankGradArgs {
  const float* margin; const float* label;
  const float* weight;                  // one per group (nullptr = 1), times wscale = groups / sum of the weights over every rank
  double wscale;
  float2* gpair; unsigned* absmax;
  int64_t n, row_offset;
  float subsample; unsigned seed; unsigned long long iter;
  int objective;                        // kRankPairwise, kRankNdcg or kRankMap
  int k;                                // lambdarank_num_pair_per_sample: the topk truncation, or the draws per document under mean
  int exp_gain, normalization, score_normalization;
  int mean;                             // lambdarank_pair_method=mean: draw k partners per document outside its label bucket
  unsigned long long pair_stream;       // mean: draw j of a document is rng_uniform(seed, pair_stream + j, row + row_offset)
};

// group_ptr empty: one group of all n rows.  Sorts the labels within the groups (the label order of IDCG).
void rank_groups_build(const std::vector<unsigned>& group_ptr, const float* label, int64_t n, RankGroups* rg, RankScratch* sc, cudaStream_t s);
void launch_rank_gradient(const RankGradArgs& a, const RankGroups& rg, RankScratch* sc, cudaStream_t s);
// ndcg (map = 0) or map (map = 1) at cutoff k (0 = the whole group) of every group, weighted by weight (one per group, nullptr = 1):
// out[0] = sum of w_g v_g, out[1] = sum of w_g (written, not added; the sums run in a fixed order)
void rank_metric(const float* margin, const float* label, const float* weight, const RankGroups& rg, int map, int k, int exp_gain, int minus,
                 RankScratch* sc, double* out, cudaStream_t s);

}  // namespace b200
