// refresh.h -- process_type=update (upstream GBTree with updater=refresh,prune): the per-node gradient sums of existing trees
// over the rows of a matrix, and the refresh / prune / compaction of each tree on the device (DESIGN.md "Refresh and prune").
#pragma once
#include "engine.h"
#include "misc.h"
#include "tree.h"

namespace b200 {

enum RefreshOp : int { kOpRefresh = 0, kOpPrune = 1 };
constexpr int kMaxRefreshOps = 8;
// a layer whose nodes fit keeps its (g_q, h_q) accumulators in shared memory (16 B per node); larger layers add into global int64
constexpr int kRefreshSmemNodes = 3072;

// The trees to update are packed one after another (node offsets node_off, absolute over every tree to update); a launch
// covers the T trees of one layer, from tree_node_off[0] = the layer's first node.
struct RefreshSumArgs {
  const float* X; int64_t n; int F;
  const DevNode* nodes;             // the trees in the predictor's node format
  const int* tree_node_off;         // [T + 1]
  const int* tree_class;            // [T] the gradient column of each tree
  int T, layer_nodes;               // layer_nodes = tree_node_off[T] - tree_node_off[0]
  const float2* gpair; int64_t gp_stride;     // [K][gp_stride] (g, h) pairs
  const float* scales;              // the round's fixed-point scales: [0] sg [1] sh
  GH64* sums;                       // by absolute node id, zero on entry for the layer; each row adds its pair to its leaf
};
void launch_refresh_sums(const RefreshSumArgs& a, cudaStream_t s);

struct RefreshTreeArgs {
  TreeArrays in;                    // the trees to update, by absolute node id
  const int* tree_node_off; int T;  // as in RefreshSumArgs
  GH64* sums;                       // leaf sums from launch_refresh_sums (all-reduced); the internal nodes' sums are derived here
  const float* scales;              // [2] 1/sg [3] 1/sh
  TrainParamDev p;                  // eta = fl(eta / num_parallel_tree)
  int ops[kMaxRefreshOps]; int nops; int refresh_leaf;
  int* scratch;                     // [3][total_nodes]: depth, parent, new id
  int64_t total_nodes;
  unsigned char* out_blocks;        // tree t's result: grow.h tree_block_layout(out_blocks + block_off[t], its input node count)
  const int64_t* block_off;         // by absolute tree id (tree t of the launch is tree first_tree + t)
  int first_tree;
  DevNode* out_nodes;               // tree t's predictor nodes at out_nodes + tree_node_off[t] - tree_node_off[0]
};
void launch_refresh_trees(const RefreshTreeArgs& a, cudaStream_t s);

}  // namespace b200
