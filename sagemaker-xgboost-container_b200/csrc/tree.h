// tree.h -- kernel argument blocks and launchers of the tree builder (see tree.cu, hist.cu, misc.cu).
#pragma once
#include "engine.h"

namespace b200 {

constexpr unsigned kPartTile = 2048;       // rows per partition tile (256 threads x 8 consecutive rows)

struct TrainParamDev {
  float eta, lambda, alpha, gamma, min_child_weight, max_delta_step;
  int max_depth, max_leaves;
};

struct EvalArgs {
  const GH64* hist_pool; GrowState gs; const int* cut_ptrs; const unsigned char* feat_mask;
  TrainParamDev p; int F, ngroups, tw, ntail, has_missing, level, max_level_nodes;
  const int* monotone;            // per-feature monotone constraint (-1, 0, +1), nullptr = none
  const unsigned char* node_allowed;   // interaction constraints: [cap_nodes][F] flags of the features a node may split on, nullptr = none
  float colsample_bynode; unsigned seed; const int* tree_index;     // per-node feature subset inside feat_mask (the level's set); tree index in device memory (graph replay)
};

struct ApplyArgs {
  GrowState gs; TreeArrays tree; const int* cut_ptrs; const float* cut_vals; const float* min_vals;
  TrainParamDev p; unsigned* scratch; int nblocks /* candidate blocks per node: groups + tail */, level, max_level_nodes, next_base, next_half;
  const int* monotone;            // as in EvalArgs
  // interaction constraints (upstream FeatureInteractionConstraintHost): per node the features used on its path and the features
  // it may split on ([cap_nodes][F] each), the constraint sets as a membership matrix [n_sets][F]
  unsigned char* node_path; unsigned char* node_allowed; const unsigned char* ic_sets; int n_ic_sets, F;
};

struct PartArgs {
  GrowState gs; TreeArrays tree; const uint8_t* bins_col; int64_t n; const unsigned* ridx_cur; unsigned* ridx_next;
  // the gradients travel with the row ids (position order): float2 (g,h) pairs, or with g_only (constant hessian, h == 1 for
  // every row) float g alone.  At the root gp_cur is the round's gradients by row, in the same layout (the dense g with g_only).
  const void* gp_cur; void* gp_next; int g_only;
  const unsigned* tl_cur; unsigned* tl_next;  // ... and so do the 4 tail bin bytes of a row (nullptr: no 4-wide tail, or it is in bins_gather)
  int has_missing, level, max_level_nodes;
  int build_only;                             // write only the child whose histogram is built (its rows are never read again otherwise)
  unsigned long long* rows_counter;           // optional (profiling): [0] += rows of split nodes read, [1] += rows written
};

// Depth-wise growth up to kRouteMaxDepth keeps one byte per row, in row order: the id of the row's current node (< 255).  Each
// level routes every row from its split byte (route_kernel), scans the tiles' row counts per built child in a fixed order
// (route_scan_kernel) and writes only the built children's rows into their segments (scatter_kernel).
constexpr int kRouteMaxDepth = 7;
constexpr unsigned kRouteTile = 2048;      // rows per route / scatter tile (256 threads x 8 rows)
constexpr int kRouteMaxNodes = 256;        // node ids of a tree of depth kRouteMaxDepth: 0 .. 254
constexpr int kRouteMaxBuild = 1 << (kRouteMaxDepth - 2);      // built children of the deepest routed level
struct RouteArgs {
  GrowState gs; TreeArrays tree; const uint8_t* bins_col; int64_t n;
  uint8_t* node_of_row;                       // [n] the tree node each row is in
  unsigned* tile_counts;                      // [kRouteMaxBuild][ntiles]: a tile's rows per built child, then their offset in it
  unsigned ntiles; int has_missing, level;
  // what scatter_kernel writes for a built row, read by ROW: g of the dense g array (g_only; constant hessian) or the class's
  // (g,h) pair, and the 4 tail bytes of a 4-wide tail (tail_row: bins_tail as words; nullptr when the tail does not travel with the ids)
  const float* g; const float2* gpair; int g_only; const unsigned* tail_row;
  unsigned* ridx; void* gp; unsigned* tl;     // the built children's rows by position
  unsigned long long* rows_counter;           // optional (profiling): [0] += rows routed, [1] += rows scattered
};

struct HistArgs {
  const uint8_t* bins;          // main: row-major [n][ngroups*32 B]
  const uint8_t* bins_tail;     // tail: row-major [n][tw B], nullptr when tw == 0
  const unsigned* tail_pos;     // tw == 4 only: the rows' tail words by POSITION (they travel with the row ids); nullptr = gather from bins_tail
  int64_t n;
  int row_stride;               // ngroups * 32
  const uint8_t* bins_gather;   // rows for the gathered passes (BinnedMatrix::bins_gather) and their stride
  int gather_stride;
  int tail_in_gather;           // gathered passes read the tail bytes from the row's own line of bins_gather (tail_pos unused)
  int tw;                       // tail width in bytes (0, 4, 8)
  const float2* gpair;          // (g, h) by POSITION in the row-id buffer (== by row at the root)
  const float* gpos;            // constant hessian: g alone by POSITION (the dense g at the root), h == 1.0f for every row (gpair
                                // unused); nullptr = gpair
  const unsigned* ridx;         // row ids by segment position; nullptr = identity (root)
  const int* build_count;       // number of nodes to build
  const int* build_nid;         // their node ids
  const unsigned* build_prefix; // exclusive prefix of their row counts, [count] = total
  const unsigned* seg_begin;    // per nid
  const int* hist_slot;         // per nid
  const float* scales;          // sg, sh
  GH64* hist_pool;              // slot stride = hist_slot_entries(ngroups, tw)
  GH64* node_sum;               // per nid, accumulated only when accumulate_sum
  // hist_gather_kernel's per-segment partial histograms: segment b of CTA x leaves its int32 {g, h} accumulators (h: the bits of
  // the unsigned H accumulator) in slot entry order at partial slot x + b, and hist_reduce_kernel adds them to the pool;
  // hist_partial_entries() entries.  B200XGB_HIST_RED_FLUSH=1 flushes with RED.ADD.64 into the pool instead.
  int2* partials;
  int ngroups;
  int ng_chunk;                 // groups per blockIdx.y chunk (set by the launcher)
  int accumulate_sum;
  int g_only;                   // constant-hessian root pass: accumulate G only from gpos (the slot already holds the cached H plane)
  int window_rows;              // rows a CTA may accumulate between two int32 overflow checks (engine.h window_rows_for)
  int force_gather;             // tests / profiling: use hist_gather_kernel even for the contiguous root pass
  unsigned long long* rows_counter;   // optional: += rows processed by this launch (profiling)
};

// grow_policy=lossguide (one expansion per iteration; tree.cu)
constexpr int kLgRootSlot = 0, kLgStageSlot = 1, kLgFirstFreeSlot = 2;     // histogram pool slots: root, all-reduce staging, then one per expansion
void launch_apply_lossguide(const ApplyArgs& a, int iter, cudaStream_t s);
void launch_lg_copy_back(const PartArgs& a, unsigned* ridx_dst, void* gp_dst, unsigned* tl_dst, unsigned max_tiles, cudaStream_t s);
void launch_zero_build_slots(const GrowState& gs, GH64* pool, size_t slot_entries, int max_build, cudaStream_t s);
void launch_lg_stage(const GrowState& gs, GH64* pool, size_t slot_entries, int to_stage, cudaStream_t s);
void launch_hist_build(const HistArgs& a, int num_sms, cudaStream_t stream);
// entries of HistArgs::partials for builds of at most max_build nodes on num_sms SMs
size_t hist_partial_entries(int ngroups, int tw, int num_sms, int max_build);
void hist_configure();     // one-time function attributes (must happen outside stream capture)
const char* hist_last_kernel();   // name of the kernel variant the last launch used (profiling / tests)
void launch_init_tree(const GrowState& gs, const TreeArrays& t, unsigned n, cudaStream_t s);   // the root's histogram: slot kLgRootSlot
void launch_scales(const GrowState& gs, int grad_bits, cudaStream_t s);
void launch_eval(const EvalArgs& a, int max_nodes_level, cudaStream_t s);
void launch_apply(const ApplyArgs& a, cudaStream_t s);
void launch_partition(const PartArgs& a, unsigned max_tiles, cudaStream_t s);
void launch_route(const RouteArgs& a, cudaStream_t s);     // route + scan + scatter of one level
// margin[:, k] += fl(*leaf_scale * leaf) of the finished tree (leaf_scale: one float on the device, 1 except under booster=dart).
// node_of_row: the node each row was routed to (the walk starts there), nullptr = walk from the root
void launch_update_margin(const TreeArrays& t, const int* n_nodes, const uint8_t* bins_col, int64_t n, int has_missing, const uint8_t* node_of_row,
                          float* margin, int K, int k, const float* leaf_scale, cudaStream_t s);
void launch_subtract(const GrowState& gs, GH64* pool, size_t slot_entries, int max_build, cudaStream_t s);

}  // namespace b200
