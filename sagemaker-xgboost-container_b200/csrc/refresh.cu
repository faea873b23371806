// refresh.cu -- process_type=update: refresh and prune existing trees (upstream src/tree/updater_refresh.cc TreeRefresher and
// src/tree/updater_prune.cc TreePruner [UPSTREAM-RECALL]), with the tree builder's exact fixed-point sums.
//
// One pass over the rows per layer (refresh_sums_kernel): each row walks each of the layer's trees on the raw float matrix with
// the predictor's rule (traverse.h) and adds its quantised (g, h) pair, rounded exactly as the histogram kernels round it, to
// its leaf's int64 accumulator.  Integer addition is associative, so the sums do not depend on launch order, CTA count or the
// number of GPUs.  Then one CTA per tree (refresh_tree_kernel) derives the internal nodes' sums bottom-up, recomputes the
// statistics with the builder's own arithmetic (split_math.h), prunes, compacts the surviving nodes and writes the tree block
// and the predictor nodes: a round needs no host synchronisation.
#include <algorithm>
#include "grow.h"
#include "refresh.h"
#include "split_math.h"
#include "traverse.h"

namespace b200 {

template <bool SMEM>
__global__ void __launch_bounds__(256) refresh_sums_kernel(RefreshSumArgs a) {
  extern __shared__ unsigned long long s_acc[];              // SMEM: [layer nodes][2] (g_q, h_q)
  const int base = a.tree_node_off[0];
  const int nl = a.tree_node_off[a.T] - base;
  if (SMEM) {
    for (int i = threadIdx.x; i < 2 * nl; i += blockDim.x) s_acc[i] = 0ull;
    __syncthreads();
  }
  unsigned long long* g_acc = reinterpret_cast<unsigned long long*>(a.sums) + 2 * (int64_t)base;
  const float sg = a.scales[0], sh = a.scales[1];
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
    const float* x = a.X + r * a.F;
    for (int t = 0; t < a.T; ++t) {
      const int off = a.tree_node_off[t];
      DevNode leaf;
      const int nid = tree_leaf(a.nodes + off, x, a.F, &leaf);
      const float2 gh = a.gpair[(int64_t)a.tree_class[t] * a.gp_stride + r];
      // the histogram kernels' rounding (hist.cu quant): g_q = rint(g * sg), h_q = rint(h * sh)
      const long long gq = (long long)__float2int_rn(gh.x * sg);
      const long long hq = (long long)(unsigned)__float2int_rn(gh.y * sh);
      const int i = off - base + nid;
      if (SMEM) { atomicAdd(&s_acc[2 * i], (unsigned long long)gq); atomicAdd(&s_acc[2 * i + 1], (unsigned long long)hq); }
      else { atomicAdd(&g_acc[2 * i], (unsigned long long)gq); atomicAdd(&g_acc[2 * i + 1], (unsigned long long)hq); }
    }
  }
  if (SMEM) {
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * nl; i += blockDim.x) if (s_acc[i]) atomicAdd(&g_acc[i], s_acc[i]);
  }
}

// One single-thread CTA per tree of the layer (a tree is at most a few thousand nodes, walked a few times in node order).
__global__ void __launch_bounds__(1) refresh_tree_kernel(RefreshTreeArgs a) {
  const int t = blockIdx.x;
  const int off = a.tree_node_off[t], nn = a.tree_node_off[t + 1] - off;
  const TrainParamDev& p = a.p;
  const TreeArrays& in = a.in;
  const TreeBlock ob = tree_block_layout(a.out_blocks + a.block_off[a.first_tree + t], (size_t)nn);
  const TreeArrays& o = ob.t;
  int* depth = a.scratch + off; int* par = a.scratch + a.total_nodes + off; int* nid_new = a.scratch + 2 * a.total_nodes + off;
  GH64* S = a.sums + off;
  for (int i = 0; i < nn; ++i) {
    const int j = off + i;
    o.left[i] = in.left[j]; o.right[i] = in.right[j]; o.parent[i] = in.parent[j]; o.split_index[i] = in.split_index[j];
    o.split_bin[i] = in.split_bin[j]; o.default_left[i] = in.default_left[j]; o.split_cond[i] = in.split_cond[j];
    o.base_weight[i] = in.base_weight[j]; o.loss_chg[i] = in.loss_chg[j]; o.sum_hess[i] = in.sum_hess[j];
    nid_new[i] = -1; depth[i] = 0; par[i] = -1;              // nid_new: 0 = alive, -1 = unreachable or deleted by the prune
  }
  // Children lie after their parent (the model reader checks it), so a forward walk from the root marks the reachable nodes and
  // sets their depths and parents, and a backward one sums them.  Slots no path reaches (upstream's deleted nodes, which the
  // legacy reader keeps as zero leaves) stay dead: no row reaches them, the prune never walks them, the compaction drops them.
  // No reachable node has two parents (begin_update checks it on the host).
  nid_new[0] = 0;
  for (int i = 0; i < nn; ++i) {
    if (nid_new[i] < 0 || o.left[i] == -1) continue;
    const int L = o.left[i], R = o.right[i];
    nid_new[L] = 0; nid_new[R] = 0; depth[L] = depth[i] + 1; depth[R] = depth[i] + 1; par[L] = i; par[R] = i;
  }
  for (int i = nn - 1; i >= 0; --i)
    if (nid_new[i] >= 0 && o.left[i] != -1) { const GH64 l = S[o.left[i]], r = S[o.right[i]]; S[i].g = l.g + r.g; S[i].h = l.h + r.h; }
  const double isg = (double)a.scales[2], ish = (double)a.scales[3];
  for (int op = 0; op < a.nops; ++op) {
    if (a.ops[op] == kOpRefresh) {
      for (int i = 0; i < nn; ++i) {
        if (nid_new[i] < 0) continue;
        const double G = (double)S[i].g * isg, H = (double)S[i].h * ish;
        const float w = calc_weight(p, G, H);
        o.sum_hess[i] = (float)H;
        if (o.left[i] == -1) {
          // the builder's leaf rule (tree.cu expand_node / finish_root): a leaf child stores fl(eta / P) * w, a root leaf w
          o.base_weight[i] = i == 0 ? w : p.eta * w;
          if (a.refresh_leaf) o.split_cond[i] = p.eta * w;
        } else {
          const int L = o.left[i], R = o.right[i];
          const double GL = (double)S[L].g * isg, HL = (double)S[L].h * ish, GR = (double)S[R].g * isg, HR = (double)S[R].h * ish;
          o.base_weight[i] = w;
          o.loss_chg[i] = calc_split_gain(p, GL, HL, GR, HR) - calc_gain(p, G, H);
        }
      }
    } else {
      // TreePruner::TryPruneLeaf for every leaf in node order: a parent of two leaves whose split gains less than gamma + kRtEps,
      // or that lies too deep, becomes a leaf of value fl(eta / P) * base_weight; then the same test one level up
      for (int i = 0; i < nn; ++i) {
        if (nid_new[i] < 0 || o.left[i] != -1) continue;
        int cur = i, d = depth[i];
        while (cur != 0) {
          const int pid = par[cur], L = o.left[pid], R = o.right[pid];
          if (o.left[L] != -1 || o.left[R] != -1) break;
          if (!(o.loss_chg[pid] < p.gamma + 1e-6f || (p.max_depth > 0 && d > p.max_depth))) break;
          nid_new[L] = -1; nid_new[R] = -1;
          o.left[pid] = -1; o.right[pid] = -1; o.split_index[pid] = 0; o.split_bin[pid] = -1; o.default_left[pid] = 0;
          o.loss_chg[pid] = 0.f; o.split_cond[pid] = p.eta * o.base_weight[pid];
          cur = pid; --d;
        }
      }
    }
  }
  // compaction: the surviving nodes in their order (parents still precede children, adjacent sibling pairs stay adjacent)
  int cnt = 0;
  for (int i = 0; i < nn; ++i) if (nid_new[i] >= 0) nid_new[i] = cnt++;
  for (int i = 0; i < nn; ++i) {
    const int j = nid_new[i];
    if (j < 0) continue;                                     // j <= i: position j has been read already
    const int L = o.left[i], R = o.right[i];
    o.left[j] = L < 0 ? -1 : nid_new[L]; o.right[j] = R < 0 ? -1 : nid_new[R];
    o.parent[j] = i == 0 ? o.parent[0] : nid_new[par[i]];
    o.split_index[j] = o.split_index[i]; o.split_bin[j] = o.split_bin[i]; o.default_left[j] = o.default_left[i];
    o.split_cond[j] = o.split_cond[i]; o.base_weight[j] = o.base_weight[i]; o.loss_chg[j] = o.loss_chg[i]; o.sum_hess[j] = o.sum_hess[i];
  }
  *ob.n_nodes = cnt;
  DevNode* nodes = a.out_nodes + (off - a.tree_node_off[0]);
  for (int j = 0; j < cnt; ++j) {
    DevNode d; d.cond = o.split_cond[j]; d.left = o.left[j]; d.right = o.right[j];
    d.fidx_dl = (unsigned)o.split_index[j] | ((unsigned)o.default_left[j] << 31);
    nodes[j] = d;
  }
}

void launch_refresh_sums(const RefreshSumArgs& a, cudaStream_t s) {
  if (a.n == 0 || a.T == 0) return;
  const int64_t blocks = std::min<int64_t>((a.n + 255) / 256, (int64_t)engine_num_sms() * 8);
  if (a.layer_nodes <= kRefreshSmemNodes) refresh_sums_kernel<true><<<(unsigned)blocks, 256, 2 * sizeof(unsigned long long) * a.layer_nodes, s>>>(a);
  else refresh_sums_kernel<false><<<(unsigned)blocks, 256, 0, s>>>(a);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

void launch_refresh_trees(const RefreshTreeArgs& a, cudaStream_t s) {
  if (a.T == 0) return;
  refresh_tree_kernel<<<a.T, 1, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
