// grow.cu -- the tree builder (grow.h): its device buffers, the launch sequence of one tree, graph capture and replay.
#include "grow.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include "comm.h"

namespace b200 {

__global__ void pack_tree_kernel(TreeArrays t, const int* n_nodes, DevNode* out, int cap) {
  const int nn = *n_nodes;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += gridDim.x * blockDim.x) {
    DevNode d;
    if (i < nn) { d.cond = t.split_cond[i]; d.left = t.left[i]; d.right = t.right[i]; d.fidx_dl = (unsigned)t.split_index[i] | ((unsigned)t.default_left[i] << 31); }
    else { d.cond = 0.f; d.left = -1; d.right = -1; d.fidx_dl = 0; }
    out[i] = d;
  }
}
// Constant-hessian root pass (reg:squarederror without weights / subsampling): the H plane of the root histogram is the
// same every round, so it is snapshotted once and later rounds start the root slot from it and accumulate G only.
__global__ void snapshot_h_kernel(const GH64* slot, long long* cache, size_t entries) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < entries; e += (size_t)gridDim.x * blockDim.x) cache[e] = slot[e].h;
}
__global__ void slot_from_cache_kernel(GH64* slot, const long long* cache, size_t entries) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < entries; e += (size_t)gridDim.x * blockDim.x) { GH64 v; v.g = 0; v.h = cache[e]; slot[e] = v; }
}
__global__ void gather_u32_kernel(const unsigned* src, const unsigned* idx, unsigned* dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

void* PinnedPool::take(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  while (cur < chunks.size() && off + bytes > chunks[cur].second) { ++cur; off = 0; }
  if (cur >= chunks.size()) { size_t sz = std::max<size_t>(bytes, 4u << 20); char* p = nullptr; CUDA_OK(cudaMallocHost(&p, sz)); chunks.emplace_back(p, sz); off = 0; }
  void* r = chunks[cur].first + off; off += bytes; return r;
}
// a 4-wide tail rides with the row ids through the partition unless the aligned row copy already holds it
static bool tail_by_position(const BinnedMatrix& bm) { return bm.tw == 4 && !bm.tail_in_gather; }

// Points the GrowState arrays into a block at `base`, in this order, and returns the block's size (the peer all-reduce maps
// the block whole).
size_t TreeBuilder::carve(GrowState& gs, uintptr_t base) const {
  const size_t N = cap_nodes, L = max_level_nodes, nblocks = ngroups + (tw > 0 ? 1 : 0);
  size_t off = 0;
  auto take = [&](auto*& p, size_t bytes) { p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off); off += (bytes + 255) & ~(size_t)255; };
  take(gs.seg_begin, 4 * N); take(gs.seg_count, 4 * N); take(gs.hist_slot, 4 * N); take(gs.node_sum, 16 * N); take(gs.root_gain, 4 * N); take(gs.weight, 4 * N);
  take(gs.best, sizeof(SplitCand) * N); take(gs.best_group, sizeof(SplitCand) * N * nblocks);
  take(gs.level_nodes, 4 * (size_t)(kMaxDepth + 1) * L); take(gs.level_count, 4 * (kMaxDepth + 2));
  take(gs.build_nid, 4 * L); take(gs.build_sub_nid, 4 * L); take(gs.build_parent_slot, 4 * L); take(gs.build_count, 4); take(gs.build_prefix, 4 * (L + 1));
  take(gs.part_action, 4 * L); take(gs.tile_prefix, 4 * (L + 1));
  take(gs.tile_desc, 8 * ((size_t)max_tiles + 1)); gs.part_ctl = (unsigned*)(gs.tile_desc + max_tiles);     // descriptors, then part_ctl
  take(gs.n_leaves, 4); take(gs.scales, 16); take(gs.absmax, 8);
  take(gs.depth, 4 * N); take(gs.open, N); take(gs.n_slots, 4); take(gs.lg_done, 4); take(gs.lower, 4 * N); take(gs.upper, 4 * N);
  return off;
}

void TreeBuilder::ensure(const BinnedMatrix& bm, int max_depth_, int K, int lg_iters_, int n_ic_) {
  const bool tail_pos_ = tail_by_position(bm);
  const int64_t stride_ = (bm.n + 63) & ~(int64_t)63;
  if (n == bm.n && F == bm.F && ngroups == bm.ngroups && tw == bm.tw && tail_pos == tail_pos_ && max_depth == max_depth_ && lg_iters == lg_iters_ &&
      n_ic == n_ic_ && gpair.n >= (size_t)stride_ * K + 512) return;
  if (lg_iters_ == 0) B200_CHECK(max_depth_ >= 1 && max_depth_ <= kMaxDepth, "max_depth must be in [1, 16] for the B200 depth-wise hist builder");
  n = bm.n; F = bm.F; ngroups = bm.ngroups; tw = bm.tw; tail_pos = tail_pos_; max_depth = max_depth_; lg_iters = lg_iters_; n_ic = n_ic_;
  gp_stride = stride_; root_h_valid = false;
  cudaStream_t s = engine_stream();
  if (peer_reduce_active()) {                     // peers still map the buffers that are about to be freed: unmap everywhere first
    peer_reduce_close();
    DevBuf<unsigned> bar; bar.alloc(1); bar.zero(s);
    Comm::get().allreduce_max_u32(bar.p, 1, s);
    Comm::get().sync_stream(s);
  }
  for (auto& tg : graphs) tg.destroy();
  size_t pool_slots; int max_nodes;
  if (lg_iters > 0) {            // lossguide: two children per expansion; "levels" 0 / 1 hold the split node and its children
    max_nodes = 2 * lg_iters + 1; max_level_nodes = 2; region = 0;
    pool_slots = (size_t)lg_iters + kLgFirstFreeSlot;         // root, staging, one fresh slot per expansion
  } else {
    max_nodes = (1 << (max_depth + 1)) - 1; max_level_nodes = 1 << (max_depth - 1); region = max_level_nodes;
    pool_slots = 2 * (size_t)region;
  }
  cap_nodes = (max_nodes + 15) & ~15;
  slot_stride = hist_slot_entries(ngroups, tw);
  const size_t partial_entries = hist_partial_entries(ngroups, tw, engine_num_sms(), max_level_nodes);
  const size_t pool_bytes = pool_slots * slot_stride * sizeof(GH64) + partial_entries * sizeof(int2);
  size_t free_b = 0, total_b = 0; cudaMemGetInfo(&free_b, &total_b);
  B200_CHECK(pool_bytes < free_b / 2 + hist_pool.n * sizeof(GH64) + hist_partials.n * sizeof(int2),
             "histogram pool for this max_depth / max_leaves / feature count does not fit in device memory");
  hist_pool.alloc(pool_slots * slot_stride);
  hist_partials.alloc(partial_entries);
  gpair.alloc((size_t)gp_stride * K + 512); gpair.zero(s); err.alloc(1); tree_index_dev.alloc(1);
  if (!leaf_scale.p) { leaf_scale.alloc(1); set_leaf_scale(1.0f); }
  root_h_cache.alloc(slot_stride);
  const bool routed = routes(lg_iters, max_depth);
  for (int i = 0; i < 2; ++i) { const size_t m = i == 0 || !routed ? (size_t)n : 0; ridx[i].alloc(m); gp[i].alloc(m); tl[i].alloc(tail_pos ? m : 0); }
  route_tiles = routed ? (unsigned)((n + kRouteTile - 1) / kRouteTile) : 0u;
  node_of_row.alloc(routed ? (size_t)n : 0);
  route_counts.alloc(routed && max_depth >= 2 ? ((size_t)1 << (max_depth - 2)) * route_tiles : 0);     // built children of the deepest routed level
  max_tiles = (unsigned)((n + kPartTile - 1) / kPartTile) + max_level_nodes + 1;
  scratch.alloc(3 * (size_t)max_level_nodes + 8);
  state_block.alloc(carve(gs, 0)); state_block.zero(s);
  carve(gs, (uintptr_t)state_block.p);
  tree_block.alloc(tree_block_bytes(cap_nodes));
  const TreeBlock tb = tree_block_layout(tree_block.p, cap_nodes);
  gs.n_nodes = tb.n_nodes; ta = tb.t; packed.alloc(cap_nodes);
  ic_path.alloc(n_ic ? (size_t)cap_nodes * F : 0); ic_allowed.alloc(n_ic ? (size_t)cap_nodes * F : 0);
  ic_sets.alloc((size_t)n_ic * F); ic_sets_host.clear();
  hist_configure();
  // multi-rank: map the peers' histogram pools / grow-state blocks over NVLink (collective; every rank gets here in its first update)
  global_n = n;
  if (Comm::get().distributed()) {
    peer_reduce_setup({{hist_pool.p, hist_pool.n * sizeof(GH64)}, {state_block.p, state_block.n}}, s);
    DevBuf<double> dsum; dsum.alloc(1); double v = (double)n;
    CUDA_OK(cudaMemcpyAsync(dsum.p, &v, sizeof v, cudaMemcpyHostToDevice, s));
    Comm::get().allreduce_sum_f64(dsum.p, 1, s);
    CUDA_OK(cudaMemcpyAsync(&v, dsum.p, sizeof v, cudaMemcpyDeviceToHost, s));
    Comm::get().sync_stream(s);
    global_n = (int64_t)v;
  }
}

float* TreeBuilder::ensure_adaptive(int targets) {
  if (adapt.ensure(n, max_leaves(), cap_nodes, targets)) for (auto& tg : graphs) tg.destroy();
  return adapt.resid.p;
}

void TreeBuilder::set_leaf_scale(float v) {
  cudaStream_t s = engine_stream();
  CUDA_OK(cudaMemcpyAsync(leaf_scale.p, &v, sizeof v, cudaMemcpyHostToDevice, s));
  Comm::get().sync_stream(s);
}

const unsigned char* TreeBuilder::upload_mask(const std::string& mask, int tree_index) {
  cudaStream_t s = engine_stream(); feat_mask.ensure(mask.size());
  CUDA_OK(cudaMemcpyAsync(feat_mask.p, mask.data(), mask.size(), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(tree_index_dev.p, &tree_index, sizeof(int), cudaMemcpyHostToDevice, s));
  Comm::get().sync_stream(s); return feat_mask.p;
}
// v into d, unless `host` says d already holds it; d is grown only when v does not fit (ensure sizes ic_sets exactly)
template <typename T> static T* upload_changed(DevBuf<T>& d, std::vector<T>& host, const std::vector<T>& v) {
  if (v == host && d.n >= v.size()) return d.p;
  cudaStream_t s = engine_stream(); d.ensure(v.size());
  CUDA_OK(cudaMemcpyAsync(d.p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, s));
  Comm::get().sync_stream(s); host = v; return d.p;
}

// padded with 0 to the feature count; uploaded again when the constraints or F change
const int* TreeBuilder::upload_monotone(const std::vector<int>& mono, int F_) {
  if (mono.empty()) return nullptr;
  B200_CHECK((int)mono.size() <= F_, "monotone_constraints has more entries than the data has features");
  std::vector<int> mh(mono); mh.resize((size_t)F_, 0);
  return upload_changed(monotone_dev, monotone_host, mh);
}
// the constraint sets as a membership matrix [n_ic][F] (ensure sized it)
void TreeBuilder::upload_interaction(const std::vector<std::vector<int>>& ic, int F_) {
  if (ic.empty()) return;
  std::vector<unsigned char> sets(ic.size() * (size_t)F_, 0);
  for (size_t si = 0; si < ic.size(); ++si)
    for (int f : ic[si]) { B200_CHECK(f < F_, "interaction_constraints names feature " + std::to_string(f) + " but the data has " + std::to_string(F_) + " features"); sets[si * F_ + f] = 1; }
  upload_changed(ic_sets, ic_sets_host, sets);
}
// The histogram pass of the root: every row in order, (g,h) of class k by row.  The deeper levels (enqueue) and the
// kernel-level entry point (debug_build_root_hist) override only the row source and their mode fields.
HistArgs TreeBuilder::hist_args(const BinnedMatrix& bm, int k) const {
  HistArgs ha{}; ha.bins = bm.bins; ha.bins_tail = bm.bins_tail; ha.n = bm.n; ha.row_stride = bm.ngroups * kSlots; ha.tw = bm.tw;
  ha.bins_gather = bm.bins_gather; ha.gather_stride = bm.gather_stride;
  ha.tail_in_gather = bm.tail_in_gather;          // gathered passes on the aligned copy always read the tail from the row's line
  ha.gpair = gpair.p + (size_t)k * gp_stride;
  ha.build_count = gs.build_count; ha.build_nid = gs.build_nid; ha.build_prefix = gs.build_prefix; ha.seg_begin = gs.seg_begin;
  ha.hist_slot = gs.hist_slot; ha.scales = gs.scales; ha.hist_pool = hist_pool.p; ha.node_sum = gs.node_sum; ha.ngroups = bm.ngroups;
  ha.partials = hist_partials.p; ha.accumulate_sum = 1; ha.window_rows = window_rows_for(global_n);
  return ha;
}

// Split evaluation of the nodes of `level` (their histograms are in the pool).  feat_mask: the level's column set or nullptr;
// a tree with column sets also samples colsample_bynode inside them.  Training (enqueue) and the kernel-level entry point
// (debug_eval_root) both start from here.
EvalArgs TreeBuilder::eval_args(const TreeInputs& in, int level, const unsigned char* feat_mask) const {
  const BinnedMatrix& bm = in.bm;
  EvalArgs ea{}; ea.hist_pool = hist_pool.p; ea.gs = gs; ea.cut_ptrs = in.cut_ptrs; ea.feat_mask = feat_mask; ea.p = in.p; ea.F = bm.F;
  ea.ngroups = bm.ngroups; ea.tw = bm.tw; ea.ntail = bm.ntail; ea.has_missing = bm.has_missing; ea.level = level; ea.max_level_nodes = max_level_nodes;
  ea.colsample_bynode = in.mask ? in.colsample_bynode : 1.0f; ea.seed = in.seed; ea.tree_index = tree_index_dev.p; ea.monotone = in.monotone;
  ea.node_allowed = in.n_ic > 0 ? ic_allowed.p : nullptr;
  return ea;
}
// Expansion of the nodes of `level`; next_base, next_half: the children's histogram slots (depth-wise).
ApplyArgs TreeBuilder::apply_args(const TreeInputs& in, int level, int next_base, int next_half) const {
  const BinnedMatrix& bm = in.bm;
  ApplyArgs aa{}; aa.gs = gs; aa.tree = ta; aa.cut_ptrs = in.cut_ptrs; aa.cut_vals = in.cut_vals; aa.min_vals = in.min_vals;
  aa.p = in.p; aa.scratch = scratch.p; aa.nblocks = bm.ngroups + (bm.tw > 0 ? 1 : 0); aa.level = level; aa.max_level_nodes = max_level_nodes;
  aa.next_base = next_base; aa.next_half = next_half; aa.monotone = in.monotone;
  if (in.n_ic > 0) { aa.node_path = ic_path.p; aa.node_allowed = ic_allowed.p; aa.ic_sets = ic_sets.p; aa.n_ic_sets = in.n_ic; aa.F = bm.F; }
  return aa;
}
// issues launch(); when profiling, brackets its launches with CUDA events and counts them
template <class Launch> void TreeBuilder::timed(ProfKind kind, Launch launch) {
  if (!profile) { launch(); return; }
  ProfEvent e; e.kind = kind; e.launches = g_kernel_launches;
  CUDA_OK(cudaEventCreate(&e.a)); CUDA_OK(cudaEventCreate(&e.b));
  CUDA_OK(cudaEventRecord(e.a, engine_stream()));
  launch();
  e.launches = g_kernel_launches - e.launches;
  CUDA_OK(cudaEventRecord(e.b, engine_stream()));
  prof_events.push_back(e);
}

constexpr int kRootRows = -1;     // the partition's input at the root: every row in order, the gradients and the tail words by row
// The fixed launch sequence of one tree (everything data dependent lives in device memory), capturable in a CUDA graph.
void TreeBuilder::enqueue(const TreeInputs& in) {
  cudaStream_t s = engine_stream();
  const BinnedMatrix& bm = in.bm;
  const int k = in.k, D = in.p.max_depth;
  const bool dist = in.world > 1;
  const int num_sms = engine_num_sms();
  launch_init_tree(gs, ta, (unsigned)bm.n, s);
  if (in.root_mode == 2) { slot_from_cache_kernel<<<num_sms, 256, 0, s>>>(hist_pool.p, root_h_cache.p, slot_stride); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
  else CUDA_OK(cudaMemsetAsync(hist_pool.p, 0, slot_stride * sizeof(GH64), s));
  // What travels with the row ids through the partition: g alone when the hessian is constant (h == 1 for every row, the
  // histograms add the constant h_q), else (g,h); plus the 4 tail bytes when the aligned row copy does not hold them.  The
  // round's gradients are then the dense g of gpair (g_dense) too, so every pass of the tree reads 4 B of gradient per row.
  const bool g_only = in.root_mode != 0;
  const int pay = g_only ? 4 : 8;
  const bool carry_tail = tail_by_position(bm);
  const bool routed = routes(in.lg_iters, D);
  if (profile && routed) {                         // route + scatter byte model per row (microbench/partition_profile.py)
    prof_part_row_bytes[0] = 3;                    // root level: split byte, node id out, node id into the scatter
    prof_part_row_bytes[1] = 4;                    // deeper levels: node id in as well
    prof_part_row_bytes[2] = pay + 4 + pay + (carry_tail ? 8 : 0);                // a built row: gradient (+ tail) by row in, id + payload (+ tail) out
  } else if (profile) {                            // partition byte model per row
    prof_part_row_bytes[0] = pay + (carry_tail ? 4 : 0) + 1;                      // root level: the gradient, tail, split byte
    prof_part_row_bytes[2] = 4 + pay + (carry_tail ? 4 : 0);                      // written: id + payload
    prof_part_row_bytes[1] = prof_part_row_bytes[2] + 1;                          // deeper levels: id + payload + split byte
  }
  // the root pass: (g,h) pairs by row; with constant hessian the dense g, through hist_gather_kernel's contiguous G-only-payload
  // mode on the snapshot tree (root_mode 1: it needs the H plane) and through hist_root_kernel<GONLY> after it (root_mode 2)
  HistArgs root = hist_args(bm, k);
  if (g_only) { root.gpair = nullptr; root.gpos = g_dense(); }
  root.g_only = in.root_mode == 2 ? 1 : 0; root.rows_counter = profile ? prof_rows.p : nullptr;
  timed(kProfRootHist, [&] { launch_hist_build(root, num_sms, s); });
  if (in.root_mode == 1) { snapshot_h_kernel<<<num_sms, 256, 0, s>>>(hist_pool.p, root_h_cache.p, slot_stride); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
  // a collective: issued directly, or (under capture) closes the current graph segment and is remembered for the replay
  auto collective = [&](std::function<void()> f) {
    if (!dist) return;
    if (!capturing) { f(); return; }
    end_segment(); capturing->colls.push_back(f);
    CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  };
  // the per-level histogram all-reduce: one NVLink peer-memory kernel inside the graph when the peers are mapped, else NCCL
  auto allreduce_hist = [&](GH64* p, size_t cnt) {
    if (!dist) return;
    if (peer_allreduce_i64(reinterpret_cast<long long*>(p), cnt, s)) return;
    collective([p, cnt, s]() { Comm::get().allreduce_sum_i64(p, cnt, s); });
  };
  allreduce_hist(hist_pool.p, slot_stride * 2);
  allreduce_hist(gs.node_sum, 2);
  if (in.n_ic > 0) {                              // root: empty path, every feature allowed
    CUDA_OK(cudaMemsetAsync(ic_path.p, 0, (size_t)bm.F, s));
    CUDA_OK(cudaMemsetAsync(ic_allowed.p, 1, (size_t)bm.F, s));
  }
  // The argument blocks of this tree's kernels, each filled in one place.  The two growth policies below pass only their own data:
  // the level, the buffer sets and the feature mask.
  auto part_args = [&](int level, int cur, int next) {                  // the partition of `level` from buffer set `cur` into set `next`
    const bool root = cur == kRootRows;
    PartArgs pa{}; pa.gs = gs; pa.tree = ta; pa.bins_col = bm.bins_col; pa.n = bm.n;
    pa.ridx_cur = root ? nullptr : ridx[cur].p; pa.ridx_next = ridx[next].p;
    const void* root_gp = g_only ? static_cast<const void*>(g_dense()) : static_cast<const void*>(gpair.p + (size_t)k * gp_stride);
    pa.gp_cur = root ? root_gp : gp[cur].p; pa.gp_next = gp[next].p; pa.g_only = g_only ? 1 : 0;
    pa.tl_cur = !carry_tail ? nullptr : (root ? reinterpret_cast<const unsigned*>(bm.bins_tail) : tl[cur].p); pa.tl_next = carry_tail ? tl[next].p : nullptr;
    pa.has_missing = bm.has_missing; pa.level = level; pa.max_level_nodes = max_level_nodes; pa.rows_counter = profile ? prof_rows.p + 2 : nullptr;
    return pa;
  };
  auto level_hist_args = [&](int set) {                                 // the build list's rows by position in buffer set `set`
    HistArgs ha = hist_args(bm, k);
    ha.ridx = ridx[set].p; ha.tail_pos = carry_tail ? tl[set].p : nullptr; ha.accumulate_sum = 0;
    ha.gpair = g_only ? nullptr : gp[set].p; ha.gpos = g_only ? reinterpret_cast<const float*>(gp[set].p) : nullptr;
    ha.rows_counter = profile ? prof_rows.p + 1 : nullptr;
    return ha;
  };
  launch_eval(eval_args(in, 0, in.mask), 1, s);
  for (int it = 0; it < in.lg_iters; ++it) {              // grow_policy=lossguide: one expansion per iteration (tree.cu apply_lossguide_kernel)
    launch_apply_lossguide(apply_args(in, 0, 0, 0), it, s);
    // live row segments always sit in buffer set 0; the partition writes the children into set 1 and they are copied straight back
    const PartArgs pa = part_args(0, it == 0 ? kRootRows : 0, 1);
    timed(kProfPartition, [&] { launch_partition(pa, max_tiles, s); });
    launch_lg_copy_back(pa, ridx[0].p, gp[0].p, tl[0].p, max_tiles, s);
    launch_zero_build_slots(gs, hist_pool.p, slot_stride, 1, s);
    timed(kProfDeepHist, [&] { launch_hist_build(level_hist_args(0), num_sms, s); });
    if (dist) {                                            // the collective needs a fixed address: go through the staging slot
      launch_lg_stage(gs, hist_pool.p, slot_stride, 1, s);
      allreduce_hist(hist_pool.p + (size_t)kLgStageSlot * slot_stride, slot_stride * 2);
      launch_lg_stage(gs, hist_pool.p, slot_stride, 0, s);
    }
    launch_subtract(gs, hist_pool.p, slot_stride, 1, s);
    launch_eval(eval_args(in, 1, nullptr), 2, s);
  }
  for (int L = 0; L < D && in.lg_iters == 0; ++L) {
    const bool final_level = (L == D - 1);
    const int next_base = ((L + 1) & 1) * region, next_half = 1 << L;
    launch_apply(apply_args(in, L, next_base, next_half), s);
    if (final_level) break;                  // children of the last level are leaves: no partition, no histograms
    if (routed) {                            // the built children's rows into buffer set 0, by row from the class's gradients
      RouteArgs ra{}; ra.gs = gs; ra.tree = ta; ra.bins_col = bm.bins_col; ra.n = bm.n; ra.node_of_row = node_of_row.p;
      ra.tile_counts = route_counts.p; ra.ntiles = route_tiles; ra.has_missing = bm.has_missing; ra.level = L;
      if (g_only) ra.g = g_dense(); else ra.gpair = gpair.p + (size_t)k * gp_stride;
      ra.g_only = g_only ? 1 : 0;
      ra.tail_row = carry_tail ? reinterpret_cast<const unsigned*>(bm.bins_tail) : nullptr;
      ra.ridx = ridx[0].p; ra.gp = gp[0].p; ra.tl = carry_tail ? tl[0].p : nullptr; ra.rows_counter = profile ? prof_rows.p + 2 : nullptr;
      timed(kProfPartition, [&] { launch_route(ra, s); });
    } else {
      PartArgs pa = part_args(L, L == 0 ? kRootRows : (L & 1) ^ 1, L & 1);     // the buffer sets alternate
      pa.build_only = L == D - 2 ? 1 : 0;                    // the next level is the last one: only the built children are read again
      timed(kProfPartition, [&] { launch_partition(pa, max_tiles, s); });
    }
    // histograms of the next level: build the smaller children, all-reduce, subtract for the siblings
    CUDA_OK(cudaMemsetAsync(hist_pool.p + (size_t)next_base * slot_stride, 0, (size_t)next_half * slot_stride * sizeof(GH64), s));
    timed(kProfDeepHist, [&] { launch_hist_build(level_hist_args(routed ? 0 : L & 1), num_sms, s); });
    allreduce_hist(hist_pool.p + (size_t)next_base * slot_stride, (size_t)next_half * slot_stride * 2);
    launch_subtract(gs, hist_pool.p, slot_stride, next_half, s);
    launch_eval(eval_args(in, L + 1, in.mask ? in.mask + (size_t)(L + 1) * bm.F : nullptr), 1 << (L + 1), s);
  }
  // the node each row was routed to (at most one split above its leaf) when the levels were routed
  const uint8_t* start = routed && D >= 2 ? node_of_row.p : nullptr;
  if (in.adaptive) {             // each leaf's value becomes fl(q * lr), q the alpha-quantile of its rows' residuals
    launch_locate_leaves(ta, gs.n_nodes, bm.bins_col, bm.n, bm.has_missing, start, g_only ? nullptr : gpair.p + (size_t)k * gp_stride, &adapt, s);
    SelectArgs sa{}; sa.values = in.resid; sa.seg = adapt.seg.p; sa.h = in.adaptive == 2 ? reinterpret_cast<const float*>(gpair.p + (size_t)k * gp_stride) + 1 : nullptr;
    sa.h_stride = 2; sa.scales = gs.scales; sa.n = bm.n; sa.nseg = max_leaves(); sa.alpha = (double)in.alpha;
    if (in.adaptive == 3) { sa.h = in.weight; sa.h_stride = 1; sa.scales = adapt.scales.p; }
    sa.leaf_nid = adapt.leaf_nid.p; sa.split_cond = ta.split_cond; sa.lr = in.p.eta;
    segmented_select(sa, &adapt, [&](unsigned long long* p, size_t cnt) { collective([p, cnt, s]() { Comm::get().allreduce_sum_i64(p, cnt, s); }); },
                     [&](unsigned* p, size_t cnt) { collective([p, cnt, s]() { Comm::get().allreduce_max_u32(p, cnt, s); }); }, s);
  }
  // prediction cache += leaf values of this tree: one row-order pass over the column-major bins
  timed(kProfMargin, [&] { launch_update_margin(ta, gs.n_nodes, bm.bins_col, bm.n, bm.has_missing, start, in.margin, in.K, k, leaf_scale.p, s); });
  if (profile) prof_margin_rows += bm.n;
  pack_tree_kernel<<<(cap_nodes + 255) / 256, 256, 0, s>>>(ta, gs.n_nodes, packed.p, cap_nodes); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
}
// ends the stream capture and appends it to the graph being captured as its next segment
void TreeBuilder::end_segment() {
  cudaGraph_t graph = nullptr; cudaGraphExec_t exec = nullptr;
  CUDA_OK(cudaStreamEndCapture(engine_stream(), &graph));
  cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  CUDA_OK(e);
  capturing->segs.push_back(exec);
}

// The sequence is replayed from a CUDA graph captured once per class and per TreeInputs: at small per-GPU shards the ~60
// launches + 6 NCCL calls per tree are otherwise CPU-launch bound.
void TreeBuilder::grow(const TreeInputs& in) {
  cudaStream_t s = engine_stream();
  static const bool no_graph = getenv("B200XGB_NO_GRAPH") != nullptr;
  if ((int)graphs.size() <= in.k) graphs.resize(in.k + 1);
  TreeGraph& tg = graphs[in.k];
  // the first tree of every class runs eagerly when ranks are connected: NCCL sets up its channels on first use
  if (profile || no_graph || (in.world > 1 && !tg.eager_done) || in.root_mode == 1) { tg.eager_done = true; enqueue(in); return; }
  if (tg.segs.empty() || memcmp(&tg.key, &in, sizeof in) != 0) {
    tg.destroy();
    const long long launches_before = g_kernel_launches;
    CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    capturing = &tg;
    try { enqueue(in); end_segment(); }
    catch (...) { capturing = nullptr; cudaGraph_t graph = nullptr; cudaStreamEndCapture(s, &graph); if (graph) cudaGraphDestroy(graph); tg.destroy(); throw; }
    capturing = nullptr;
    tg.key = in; tg.launches = g_kernel_launches - launches_before;
    g_kernel_launches = launches_before;               // capture enqueued nothing
  }
  for (size_t i = 0; i < tg.segs.size(); ++i) {
    CUDA_OK(cudaGraphLaunch(tg.segs[i], s));
    if (i < tg.colls.size()) tg.colls[i]();
  }
  g_kernel_launches += tg.launches;
}
PendingTree TreeBuilder::stage_tree() {
  cudaStream_t s = engine_stream();
  PendingTree pt; pt.cap_nodes = (size_t)cap_nodes; pt.staging = pinned.take(tree_block.n);
  if (!free_events.empty()) { pt.ready = free_events.back(); free_events.pop_back(); }
  else CUDA_OK(cudaEventCreateWithFlags(&pt.ready, cudaEventDisableTiming));
  CUDA_OK(cudaMemcpyAsync(pt.staging, tree_block.p, tree_block.n, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaEventRecord(pt.ready, s));
  return pt;
}

// Kernel-level entry point for parity tests and the roofline bench: build the histogram of all rows (or of the row
// subset `row_ids`, gradient pairs by position) from host gradient pairs `repeats` times; returns the int64 histogram in
// pool layout ([ngroups][256][32]{g,h} then the tail [256][tw]{g,h}) and the fixed-point scales.
void TreeBuilder::debug_build_root_hist(const BinnedMatrix& bm, const float* gpair_host, std::vector<long long>* hist_out, float* scales_out,
                                        int repeats, float* ms_out, int mode, const unsigned* row_ids, int64_t n_ids) {
  cudaStream_t s = engine_stream();
  const int64_t rows = row_ids ? n_ids : bm.n;
  B200_CHECK(rows <= bm.n, "debug_build_root_hist: more row ids than rows");
  CUDA_OK(cudaMemcpyAsync(gpair.p, gpair_host, sizeof(float2) * rows, cudaMemcpyHostToDevice, s));
  if (row_ids) CUDA_OK(cudaMemcpyAsync(ridx[0].p, row_ids, sizeof(unsigned) * rows, cudaMemcpyHostToDevice, s));
  // scales from max|g|, max h of the supplied pairs
  float mg = 0.f, mh = 0.f;
  for (int64_t i = 0; i < rows; ++i) { mg = std::max(mg, std::fabs(gpair_host[2 * i])); mh = std::max(mh, gpair_host[2 * i + 1]); }
  unsigned am[2]; memcpy(&am[0], &mg, 4); memcpy(&am[1], &mh, 4);
  CUDA_OK(cudaMemcpyAsync(gs.absmax, am, 8, cudaMemcpyHostToDevice, s));
  launch_scales(gs, grad_bits_for(global_n), s);
  HistArgs ha = hist_args(bm, 0);                 // the training path's arguments; the row ids and the mode bits override
  ha.ridx = row_ids ? ridx[0].p : nullptr;
  ha.force_gather = (mode & 3) == 1 ? 1 : 0; ha.g_only = (mode & 3) == 2 ? 1 : 0;
  if ((mode & 8) || ha.g_only) {                // G-only payload: g alone, h == 1.0f for every row (the supplied h is ignored)
    std::vector<float> gh((size_t)rows);
    for (int64_t i = 0; i < rows; ++i) gh[i] = gpair_host[2 * i];
    // by position after a partition; at the root the dense g of constant-hessian training, whose allocation covers whole root tiles
    float* gpos = row_ids ? reinterpret_cast<float*>(gp[0].p) : g_dense();
    if (rows) CUDA_OK(cudaMemcpyAsync(gpos, gh.data(), sizeof(float) * rows, cudaMemcpyHostToDevice, s));
    Comm::get().sync_stream(s);
    ha.gpos = gpos; ha.gpair = nullptr;
  }
  if ((mode & 4) && row_ids && tail_by_position(bm)) {     // the training path's variant: the rows' tail words by POSITION (as after a partition)
    gather_u32_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(reinterpret_cast<const unsigned*>(bm.bins_tail), ridx[0].p, tl[0].p, rows); ++g_kernel_launches;
    CUDA_OK(cudaGetLastError());
    ha.tail_pos = tl[0].p;
  }
  root_h_valid = false;                         // the debug entry point overwrites gpair and the root slot
  cudaEvent_t e0, e1; CUDA_OK(cudaEventCreate(&e0)); CUDA_OK(cudaEventCreate(&e1));
  float total = 0.f;
  for (int r = 0; r < std::max(1, repeats); ++r) {
    launch_init_tree(gs, ta, (unsigned)rows, s);
    CUDA_OK(cudaMemsetAsync(hist_pool.p, 0, slot_stride * sizeof(GH64), s));
    CUDA_OK(cudaEventRecord(e0, s));
    launch_hist_build(ha, engine_num_sms(), s);
    CUDA_OK(cudaEventRecord(e1, s));
    CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0; CUDA_OK(cudaEventElapsedTime(&ms, e0, e1)); total += ms;
  }
  if (ms_out) *ms_out = total / std::max(1, repeats);
  hist_out->resize(slot_stride * 2);
  CUDA_OK(cudaMemcpyAsync(hist_out->data(), hist_pool.p, sizeof(GH64) * slot_stride, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(scales_out, gs.scales, 4 * sizeof(float), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
}

// Kernel-level entry point for split evaluation: the root of a tree whose histogram is hist_fm ([F][256]{g,h}, int64 fixed point)
// with node totals (G, H) on the grid that launch_scales derives from max_g, max_h for the matrix's row count; lower / upper
// bound the root's weight (monotone constraints).  Runs init_tree, eval_kernel at level 0 and the expansion of the growth policy
// with the training path's arguments, and returns JSON (floats as uint32 bits).
std::string TreeBuilder::debug_eval_root(const TreeInputs& in, const long long* hist_fm, long long G, long long H, float max_g, float max_h,
                                         float lower, float upper) {
  cudaStream_t s = engine_stream();
  root_h_valid = false;                         // the root slot is overwritten
  const BinnedMatrix& bm = in.bm;
  const int F_ = bm.F;
  // the histogram in pool layout: [group][bin][slot] then the tail [bin][tw]
  std::vector<GH64> slot(slot_stride, GH64{0, 0});
  const size_t W = (size_t)bm.ngroups * kSlots, tail0 = (size_t)bm.ngroups * kGroupEntries;
  for (int f = 0; f < F_; ++f)
    for (int b = 0; b < kBins; ++b) {
      const size_t e = (size_t)f < W ? ((size_t)(f / kSlots) * kBins + b) * kSlots + f % kSlots : tail0 + (size_t)b * bm.tw + (f - W);
      slot[e].g = hist_fm[((size_t)f * kBins + b) * 2]; slot[e].h = hist_fm[((size_t)f * kBins + b) * 2 + 1];
    }
  launch_init_tree(gs, ta, (unsigned)bm.n, s);
  CUDA_OK(cudaMemcpyAsync(hist_pool.p, slot.data(), sizeof(GH64) * slot_stride, cudaMemcpyHostToDevice, s));
  const GH64 tot{G, H};
  CUDA_OK(cudaMemcpyAsync(gs.node_sum, &tot, sizeof tot, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(gs.lower, &lower, 4, cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(gs.upper, &upper, 4, cudaMemcpyHostToDevice, s));
  unsigned am[2]; memcpy(&am[0], &max_g, 4); memcpy(&am[1], &max_h, 4);
  CUDA_OK(cudaMemcpyAsync(gs.absmax, am, 8, cudaMemcpyHostToDevice, s));
  launch_scales(gs, grad_bits_for(global_n), s);
  launch_eval(eval_args(in, 0, in.mask), 1, s);
  const ApplyArgs aa = apply_args(in, 0, region, 1);
  if (in.lg_iters > 0) launch_apply_lossguide(aa, 0, s); else launch_apply(aa, s);
  // read back
  const int nblocks = bm.ngroups + (bm.tw > 0 ? 1 : 0);
  std::vector<unsigned char> sb(state_block.n), tb(tree_block.n);
  CUDA_OK(cudaMemcpyAsync(sb.data(), state_block.p, sb.size(), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(tb.data(), tree_block.p, tb.size(), cudaMemcpyDeviceToHost, s));
  Comm::get().sync_stream(s);
  GrowState h; carve(h, (uintptr_t)sb.data());
  auto bits = [](float v) { unsigned u; memcpy(&u, &v, 4); return std::to_string(u); };
  auto cand = [&](const SplitCand& c) {
    return "{\"loss_chg\":" + bits(c.loss_chg) + ",\"feature\":" + std::to_string(c.feature) + ",\"bin\":" + std::to_string(c.bin) + ",\"dleft\":" +
           std::to_string(c.dleft) + ",\"ord\":" + std::to_string(c.ord) + ",\"GL\":" + std::to_string(c.GL) + ",\"HL\":" + std::to_string(c.HL) + "}";
  };
  const TreeBlock t = tree_block_layout(tb.data(), cap_nodes);
  const int nn = *t.n_nodes;
  std::string o = "{\"scales\":[";
  for (int i = 0; i < 4; ++i) o += (i ? "," : "") + bits(h.scales[i]);
  o += "],\"root_gain\":" + bits(h.root_gain[0]) + ",\"weight\":" + bits(h.weight[0]) + ",\"best_group\":[";
  for (int i = 0; i < nblocks; ++i) o += (i ? "," : "") + cand(h.best_group[i]);
  o += "],\"best\":" + cand(h.best[0]) + ",\"n_nodes\":" + std::to_string(nn) + ",\"expanded\":" + (nn == 3 ? "true" : "false") + ",\"tree\":{";
  const char* iname[5] = {"left", "right", "parent", "split_index", "split_bin"};
  const int* iarr[5] = {t.t.left, t.t.right, t.t.parent, t.t.split_index, t.t.split_bin};
  const char* fname[4] = {"split_cond", "base_weight", "loss_chg", "sum_hess"};
  const float* farr[4] = {t.t.split_cond, t.t.base_weight, t.t.loss_chg, t.t.sum_hess};
  for (int a = 0; a < 5; ++a) { o += std::string(a ? "," : "") + "\"" + iname[a] + "\":["; for (int i = 0; i < nn; ++i) o += (i ? "," : "") + std::to_string(iarr[a][i]); o += "]"; }
  for (int a = 0; a < 4; ++a) { o += std::string(",\"") + fname[a] + "\":["; for (int i = 0; i < nn; ++i) o += (i ? "," : "") + bits(farr[a][i]); o += "]"; }
  o += ",\"default_left\":["; for (int i = 0; i < nn; ++i) o += (i ? "," : "") + std::to_string((int)t.t.default_left[i]); o += "]}";
  o += ",\"children\":[";
  for (int c = 1; c < nn && c < 3; ++c)
    o += std::string(c > 1 ? "," : "") + "{\"G\":" + std::to_string(h.node_sum[c].g) + ",\"H\":" + std::to_string(h.node_sum[c].h) + ",\"lower\":" + bits(h.lower[c]) + ",\"upper\":" + bits(h.upper[c]) + "}";
  o += "]}";
  return o;
}

void TreeBuilder::set_profile(bool on) {
  profile = on;
  if (on) { prof_rows.alloc(4); prof_rows.zero(engine_stream()); prof_margin_rows = 0; }
  for (auto& e : prof_events) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  prof_events.clear();
}
std::string TreeBuilder::profile_json() {
  cudaStream_t s = engine_stream();
  Comm::get().sync_stream(s);
  double ms[kProfKinds] = {}; long long launches[kProfKinds] = {};
  for (auto& e : prof_events) { float t = 0; CUDA_OK(cudaEventElapsedTime(&t, e.a, e.b)); ms[e.kind] += t; launches[e.kind] += e.launches; }
  unsigned long long rows[4] = {0, 0, 0, 0};
  if (prof_rows.p) CUDA_OK(cudaMemcpy(rows, prof_rows.p, sizeof rows, cudaMemcpyDeviceToHost));
  char buf[1024];
  snprintf(buf, sizeof buf, "{\"root_hist_ms\":%.6f,\"root_hist_launches\":%lld,\"root_hist_rows\":%llu,\"deep_hist_ms\":%.6f,\"deep_hist_launches\":%lld,\"deep_hist_rows\":%llu,"
           "\"part_ms\":%.6f,\"part_launches\":%lld,\"part_rows\":%llu,\"part_rows_written\":%llu,"
           "\"part_row_bytes_in_root\":%d,\"part_row_bytes_in\":%d,\"part_row_bytes_out\":%d,\"margin_ms\":%.6f,\"margin_launches\":%lld,\"margin_rows\":%lld}",
           ms[kProfRootHist], launches[kProfRootHist], rows[0], ms[kProfDeepHist], launches[kProfDeepHist], rows[1],
           ms[kProfPartition], launches[kProfPartition], rows[2], rows[3], prof_part_row_bytes[0], prof_part_row_bytes[1], prof_part_row_bytes[2],
           ms[kProfMargin], launches[kProfMargin], prof_margin_rows);
  return buf;
}

}  // namespace b200
