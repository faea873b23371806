// grow.h -- the tree builder: the device buffers of tree growth and the launch sequence of one tree, issued directly or
// replayed from CUDA graphs (DESIGN.md §4, §5).
#pragma once
#include <functional>
#include <string>
#include <type_traits>
#include <vector>
#include "adaptive.h"
#include "engine.h"
#include "misc.h"
#include "tree.h"

namespace b200 {

// Everything the launch sequence of one tree reads that is not one of the builder's own buffers.  It is also the key of the
// graph replay: a captured tree replays only for inputs equal byte for byte (there are no padding bytes) to the captured ones.
struct TreeInputs {
  BinnedMatrix bm;                        // the training matrix
  const int* cut_ptrs; const float* cut_vals; const float* min_vals;
  float* margin;                          // prediction cache [n][K]: the tree adds its leaf values to column k
  const unsigned char* mask;              // column sampling: the levels' feature sets [max_depth][F]; nullptr = every feature
  const int* monotone;                    // per-feature monotone constraints on the device, nullptr = none
  TrainParamDev p;
  float colsample_bynode; unsigned seed;
  int lg_iters, n_ic;                     // grow_policy=lossguide: expansions per tree (0 = depthwise); interaction constraint sets
  int K, k, world;                        // classes, the class of this tree, ranks of the job
  int root_mode;                          // 0 = accumulate G and H, 1 = G and H + snapshot of the root H plane, 2 = G only on top of it
  // reg:absoluteerror / reg:quantileerror: the round's residuals fl(y - m) by row of this tree's output, and the leaf refresh
  // after the structure is final (adaptive.h): 0 = none, 1 = alpha-quantile of the rows' residuals by count, 2 = by h_q
  // (weighted data), 3 = by the instance weights `weight` on their own grid (adapt.scales[1], adaptive.h weight_grid): weighted
  // data under gradient-based sampling, whose h is w / p.  alpha: 0.5 for absolute error, the target's quantile_alpha entry.
  const float* resid; const float* weight;
  int adaptive;
  float alpha;
};
static_assert(std::is_trivially_copyable<TreeInputs>::value, "TreeInputs is compared as bytes");
static_assert(sizeof(BinnedMatrix) == 4 * sizeof(void*) + sizeof(int64_t) + 8 * sizeof(int), "BinnedMatrix has padding bytes");
static_assert(sizeof(TrainParamDev) == 8 * 4, "TrainParamDev has padding bytes");
static_assert(sizeof(TreeInputs) == sizeof(BinnedMatrix) + 8 * sizeof(void*) + sizeof(TrainParamDev) + 10 * 4, "TreeInputs has padding bytes");

// The tree block, copied to the host in one piece: the node count (padded to 64 B), then `cap` entries each of left, right,
// parent, split_index, split_bin (int), split_cond, base_weight, loss_chg, sum_hess (float) and default_left (u8).
inline size_t tree_block_bytes(size_t cap) { return 64 + 9 * 4 * cap + cap; }
struct TreeBlock { int* n_nodes; TreeArrays t; };
__host__ __device__ inline TreeBlock tree_block_layout(void* base, size_t cap) {     // the tree refresh writes blocks on the device
  int* ip = (int*)((unsigned char*)base + 64); float* fp = (float*)(ip + 5 * cap);
  return {(int*)base, {ip, ip + cap, ip + 2 * cap, ip + 3 * cap, ip + 4 * cap, (unsigned char*)(fp + 4 * cap), fp, fp + cap, fp + 2 * cap, fp + 3 * cap}};
}

struct PendingTree {            // a tree still on its way from the device (async copy of its tree block into pinned memory)
  void* staging = nullptr; size_t cap_nodes = 0; cudaEvent_t ready = nullptr;
};
struct PinnedPool {
  std::vector<std::pair<char*, size_t>> chunks; size_t cur = 0, off = 0;
  ~PinnedPool() { for (auto& c : chunks) cudaFreeHost(c.first); }
  void* take(size_t bytes);
  void reset() { cur = 0; off = 0; }
};

// The per-tree launch sequence as CUDA graphs.  On one GPU it is a single graph; with NCCL it is cut into SEGMENTS at every
// collective (root + one per level): the segments are replayed as graphs and the all-reduces are issued between them as
// ordinary stream operations, so no NCCL call is ever captured (a capture with lazily connecting NCCL channels hung an
// 8-rank run in round 1) while a tree still costs ~2 host operations per level instead of ~13.
struct TreeGraph {
  std::vector<cudaGraphExec_t> segs; std::vector<std::function<void()>> colls;      // colls[i] runs after segs[i]
  TreeInputs key{}; long long launches = 0;
  bool eager_done = false;                 // a tree of this class was issued directly
  TreeGraph() = default; TreeGraph(TreeGraph&&) = default;
  ~TreeGraph() { destroy(); }
  void destroy() { for (auto e : segs) if (e) cudaGraphExecDestroy(e); segs.clear(); colls.clear(); }
};

// The tree builder.  Its own buffers are (re)allocated only in ensure, which destroys every captured graph: a graph bakes in
// their addresses, and all else it reads comes from TreeInputs.
struct TreeBuilder {
  int64_t n = 0; int F = 0, ngroups = 0, tw = 0, max_depth = 0, cap_nodes = 0, max_level_nodes = 0, region = 0; bool tail_pos = false;
  int lg_iters = 0, n_ic = 0;              // as in TreeInputs
  size_t slot_stride = 0;                  // GH64 entries per histogram slot
  int64_t gp_stride = 0;                   // rows reserved per class in gpair
  unsigned max_tiles = 0;                  // partition tiles of a level, worst case
  // rows of the whole job (sum over ranks, all-reduced once): ranks must agree on the fixed-point grid, so it follows this
  // count and N ranks and one GPU train bit-identical models on the same data
  int64_t global_n = 0;
  DevBuf<long long> root_h_cache; uint64_t root_h_uid = 0, root_h_version = 0; bool root_h_valid = false;
  GrowState gs{}; TreeArrays ta{};
  DevBuf<unsigned char> state_block;       // all GrowState arrays
  DevBuf<unsigned char> tree_block;        // tree_block_layout()
  // the partition's two buffer sets: row ids, the gradients (float g alone in the first n floats for constant-hessian objectives)
  // and the 4 tail bytes of each row, by position.  Routed growth (routes()) writes only set 0; set 1 exists only without it.
  DevBuf<GH64> hist_pool; DevBuf<unsigned> ridx[2], scratch;
  DevBuf<int2> hist_partials;              // the gathered histogram passes' per-segment partials (tree.h HistArgs::partials)
  // gpair: the round's gradients by row, [K][gp_stride] (g,h) pairs, or for constant-hessian growth (TreeInputs root_mode != 0,
  // K == 1) a dense float g[gp_stride] in the same allocation (g_dense)
  DevBuf<float2> gpair, gp[2]; DevBuf<unsigned> tl[2]; DevBuf<int> err, tree_index_dev; DevBuf<unsigned char> ic_path, ic_allowed, ic_sets;
  // routed growth: the node each row is in (row order) and the route tiles' row counts per built child (tree.h RouteArgs)
  DevBuf<uint8_t> node_of_row; DevBuf<unsigned> route_counts; unsigned route_tiles = 0;
  DevBuf<DevNode> packed;                  // the finished tree in the predictor's node format
  // the factor of the tree's leaves in the prediction cache (booster=dart: the new trees' weight, else 1).  A buffer of the
  // builder, not a TreeInputs field: a different weight every round must not force a fresh graph capture.
  DevBuf<float> leaf_scale;
  // uploaded per tree; their addresses are part of TreeInputs
  DevBuf<unsigned char> feat_mask; DevBuf<int> monotone_dev;
  std::vector<unsigned char> ic_sets_host; // what ic_sets holds
  std::vector<int> monotone_host;          // what monotone_dev holds
  PinnedPool pinned; std::vector<cudaEvent_t> free_events;
  std::vector<TreeGraph> graphs;           // per class
  TreeGraph* capturing = nullptr;          // set while enqueue runs under stream capture: collectives cut the capture
  // reg:absoluteerror / reg:quantileerror: the round's residuals and the leaf refresh's buffers, allocated by ensure_adaptive
  // (only for those objectives)
  SelectScratch adapt;
  int max_leaves() const { return lg_iters > 0 ? lg_iters + 1 : 1 << max_depth; }
  // sizes `adapt` for this builder and `targets` residual columns of n rows (destroys the captured graphs when a buffer moves);
  // the residual buffer
  float* ensure_adaptive(int targets = 1);
  // profiling: CUDA events around the launches of each kind and the partition's byte model
  enum ProfKind { kProfRootHist, kProfDeepHist, kProfPartition, kProfMargin, kProfKinds };
  struct ProfEvent { cudaEvent_t a, b; int kind; long long launches; };
  bool profile = false; std::vector<ProfEvent> prof_events;
  // [0] rows through root launches, [1] rows through deeper launches, [2] rows of split nodes read by the partition (routed:
  // rows routed), [3] rows the partition wrote (routed: built rows scattered)
  DevBuf<unsigned long long> prof_rows;
  long long prof_margin_rows = 0;
  // partition byte model per row of the last profiled tree: [0] read at the root level (no row id), [1] read at deeper levels,
  // [2] written (row id + gradient payload + tail bytes when they travel with the ids; routed: plus what a built row reads by row)
  int prof_part_row_bytes[3] = {0, 0, 0};

  ~TreeBuilder() { for (auto e : free_events) cudaEventDestroy(e); for (auto& e : prof_events) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); } }
  void ensure(const BinnedMatrix& bm, int max_depth, int K, int lg_iters, int n_ic);
  // Depth-wise trees up to kRouteMaxDepth keep a node id per row and write only the built children's rows per level (node ids
  // fit a byte); loss-guided growth expands one node at a time and deeper trees have too many built children per level, so
  // both move the rows of every split node through part_kernel.
  static bool routes(int lg_iters, int max_depth) { return lg_iters == 0 && max_depth <= kRouteMaxDepth; }
  // uploads outside the launch sequence: the tree's column sets and its index (colsample_bynode draws from it), the constraints
  const unsigned char* upload_mask(const std::string& mask, int tree_index);
  const int* upload_monotone(const std::vector<int>& mono, int F);    // nullptr when there are none
  void upload_interaction(const std::vector<std::vector<int>>& sets, int F);
  void set_leaf_scale(float v);            // for the trees grown next
  void grow(const TreeInputs& in);         // one tree into packed / tree_block: issued directly or replayed from a graph
  PendingTree stage_tree();                // async copy of the finished tree block into pinned memory
  void set_profile(bool on); std::string profile_json();
  void debug_build_root_hist(const BinnedMatrix& bm, const float* gpair_host, std::vector<long long>* hist_out, float* scales_out,
                             int repeats, float* ms_out, int mode, const unsigned* row_ids, int64_t n_ids);
  std::string debug_eval_root(const TreeInputs& in, const long long* hist_fm, long long G, long long H, float max_g, float max_h,
                              float lower, float upper);

 private:
  size_t carve(GrowState& g, uintptr_t base) const;
  void enqueue(const TreeInputs& in);
  void end_segment();
  HistArgs hist_args(const BinnedMatrix& bm, int k) const;
  float* g_dense() const { return reinterpret_cast<float*>(gpair.p); }
  EvalArgs eval_args(const TreeInputs& in, int level, const unsigned char* feat_mask) const;
  ApplyArgs apply_args(const TreeInputs& in, int level, int next_base, int next_half) const;
  template <class Launch> void timed(ProfKind kind, Launch launch);
};

}  // namespace b200
