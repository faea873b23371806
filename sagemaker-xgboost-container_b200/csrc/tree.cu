// tree.cu -- split evaluation, node expansion, sibling subtraction and row partition kernels of the
// depth-wise hist tree builder (SURVEY.md section 8a rows A9, A10, A11).  Mirrors the behaviour of upstream
// xgboost's src/tree/hist/evaluate_splits.h, src/tree/driver.h, src/tree/updater_quantile_hist.cc and
// src/common/partition_builder.h as restated in oracle/gbt_oracle.c; all control flow stays on the device.
#include <type_traits>
#include "engine.h"
#include "rng.h"
#include "tree.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// split arithmetic (float/double mix follows upstream src/tree/param.h + split_evaluator.h)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double threshold_l1(double w, double alpha) {
  if (w > +alpha) return w - alpha;
  if (w < -alpha) return w + alpha;
  return 0.0;
}
__device__ __forceinline__ float calc_weight(const TrainParamDev& p, double G, double H) {
  if (H < p.min_child_weight || H <= 0.0) return 0.0f;
  double dw = -threshold_l1(G, p.alpha) / (H + p.lambda);
  if (p.max_delta_step != 0.0f && fabs(dw) > p.max_delta_step) dw = copysign((double)p.max_delta_step, dw);
  return (float)dw;
}
// -(2 g w + (h + lambda) w^2) in float with every product rounded before the add, as upstream's CPU code evaluates it: a fused
// multiply-add would change the last bits of loss_chg, and at near-ties which split wins
__device__ __forceinline__ float gain_at_weight_f(float g, float h, float lambda, float w) {
  return -__fadd_rn(__fmul_rn(__fmul_rn(2.0f, g), w), __fmul_rn(__fmul_rn(__fadd_rn(h, lambda), w), w));
}
__device__ __forceinline__ float calc_gain_given_weight(const TrainParamDev& p, double G, double H, float w) {
  if (H <= 0.0) return 0.0f;
  if (p.max_delta_step == 0.0f) { double t = threshold_l1(G, p.alpha); return (float)(t * t / (H + p.lambda)); }
  return gain_at_weight_f((float)G, (float)H, p.lambda, w);
}
__device__ __forceinline__ float calc_gain(const TrainParamDev& p, double G, double H) {
  return calc_gain_given_weight(p, G, H, calc_weight(p, G, H));
}
__device__ __forceinline__ float calc_split_gain(const TrainParamDev& p, double GL, double HL, double GR, double HR) {
  float wl = calc_weight(p, GL, HL), wr = calc_weight(p, GR, HR);
  return calc_gain_given_weight(p, GL, HL, wl) + calc_gain_given_weight(p, GR, HR, wr);
}

// Interaction constraints (upstream src/tree/constraints.cc FeatureInteractionConstraintHost::SplitImpl [UPSTREAM-RECALL]): a
// child may split on the features already used on its path, plus every feature of each constraint set that contains ALL of the
// path's features; the root may use any feature.
__device__ __forceinline__ void interaction_children(const ApplyArgs& a, int nid, int f, int Lc, int Rc) {
  if (a.node_allowed == nullptr) return;
  const size_t F = (size_t)a.F;
  unsigned char* pl = a.node_path + (size_t)Lc * F; unsigned char* pr = a.node_path + (size_t)Rc * F;
  unsigned char* al = a.node_allowed + (size_t)Lc * F; unsigned char* ar = a.node_allowed + (size_t)Rc * F;
  const unsigned char* pp = a.node_path + (size_t)nid * F;
  for (int j = 0; j < a.F; ++j) { const unsigned char v = (pp[j] || j == f) ? 1 : 0; pl[j] = v; pr[j] = v; al[j] = v; ar[j] = v; }
  for (int s = 0; s < a.n_ic_sets; ++s) {
    const unsigned char* set = a.ic_sets + (size_t)s * F;
    bool relevant = true;
    for (int j = 0; j < a.F && relevant; ++j) if (pl[j] && !set[j]) relevant = false;
    if (relevant) for (int j = 0; j < a.F; ++j) if (set[j]) { al[j] = 1; ar[j] = 1; }
  }
}

// Monotone constraints (upstream src/tree/split_evaluator.h TreeEvaluator): weights are clamped to the node's [lower, upper]
// interval, the gain is evaluated AT the clamped weights (always the general form, never the t^2 / (H + lambda) shortcut), a
// candidate whose child weights violate the feature's constraint is rejected, and a split hands mid = (wl + wr) / 2 down to the
// children as the new bound on the constrained side.
__device__ __forceinline__ float clamp_weight(float w, float lo, float hi) { return w < lo ? lo : (w > hi ? hi : w); }
__device__ __forceinline__ float gain_at_weight(const TrainParamDev& p, double G, double H, float w) {
  if (H <= 0.0) return 0.0f;
  return gain_at_weight_f((float)G, (float)H, p.lambda, w);
}
// gain of a candidate under constraints; returns false when it violates the feature's constraint c
__device__ __forceinline__ bool constrained_split_gain(const TrainParamDev& p, double GL, double HL, double GR, double HR, float lo, float hi, int c, float* gain) {
  const float wl = clamp_weight(calc_weight(p, GL, HL), lo, hi), wr = clamp_weight(calc_weight(p, GR, HR), lo, hi);
  *gain = gain_at_weight(p, GL, HL, wl) + gain_at_weight(p, GR, HR, wr);
  return c == 0 || (c > 0 ? wl <= wr : wl >= wr);
}

// Total order of candidates == upstream SplitEntry::NeedReplace: larger loss_chg, then lower feature,
// then earlier position in scan order (forward bins ascending, then backward bins descending).
// Key: 32 bits of loss | 23 bits of inverted feature | 9 bits of inverted ord (ord < 512); features below kMaxSplitFeatures.
__device__ __forceinline__ unsigned long long cand_key(float loss, int f, int ord) {
  if (!(loss > 0.0f) || isinf(loss)) return 0ull;
  return ((unsigned long long)__float_as_uint(loss) << 32) | ((unsigned long long)(0x7FFFFFu - (unsigned)f) << 9) |
         (unsigned long long)(0x1FFu - (unsigned)ord);
}

// ---------------------------------------------------------------------------------------------
__global__ void init_tree_kernel(GrowState gs, TreeArrays t, unsigned n) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  *gs.n_nodes = 1; *gs.n_leaves = 1;
  *gs.n_slots = kLgFirstFreeSlot; *gs.lg_done = 0; gs.depth[0] = 0; gs.open[0] = 0;
  gs.lower[0] = -INFINITY; gs.upper[0] = INFINITY;
  for (int d = 0; d < kMaxDepth + 2; ++d) gs.level_count[d] = 0;
  gs.level_count[0] = 1; gs.level_nodes[0] = 0;
  gs.seg_begin[0] = 0; gs.seg_count[0] = n; gs.hist_slot[0] = kLgRootSlot;
  gs.node_sum[0].g = 0; gs.node_sum[0].h = 0;
  *gs.build_count = 1; gs.build_nid[0] = 0; gs.build_sub_nid[0] = -1; gs.build_parent_slot[0] = -1;
  gs.build_prefix[0] = 0; gs.build_prefix[1] = n;
  t.left[0] = -1; t.right[0] = -1; t.parent[0] = 2147483647; t.split_index[0] = 0; t.split_bin[0] = -1;
  t.default_left[0] = 0; t.split_cond[0] = 0.f; t.base_weight[0] = 0.f; t.loss_chg[0] = 0.f; t.sum_hess[0] = 0.f;
}

// Fixed-point scales from the all-reduced max|g|, max h of this round: power-of-two so that
// quantisation is pure rounding to a binary grid and the inverse scaling is exact.
__global__ void scales_kernel(GrowState gs, int grad_bits) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float mg = __uint_as_float(gs.absmax[0]), mh = __uint_as_float(gs.absmax[1]);
  int eg = 0, eh = 0;
  if (mg > 0.f && isfinite(mg)) frexpf(mg, &eg);     // mg < 2^eg
  if (mh > 0.f && isfinite(mh)) frexpf(mh, &eh);
  float sg = ldexpf(1.0f, grad_bits - eg), sh = ldexpf(1.0f, grad_bits + 1 - eh);
  gs.scales[0] = sg; gs.scales[1] = sh; gs.scales[2] = 1.0f / sg; gs.scales[3] = 1.0f / sh;
}

// ---------------------------------------------------------------------------------------------
// split evaluation: one block per (alive node of the level, feature group); thread = (slot, 8-bin segment).
// The kernel is a latency chain (per candidate: int64 prefix, four double divisions), not a throughput problem: 32 segments
// of 8 bins instead of 8 of 32 cut it from 33 us to ~10 us per launch, which matters at 8 GPUs where it does not shrink.
// ---------------------------------------------------------------------------------------------
constexpr int kEvalSegs = 32, kEvalBinsPerSeg = kBins / kEvalSegs;
__global__ void __launch_bounds__(32 * kEvalSegs) eval_kernel(EvalArgs a) {
  const int li = blockIdx.x;
  if (li >= a.gs.level_count[a.level]) return;
  const int nid = a.gs.level_nodes[(size_t)a.level * a.max_level_nodes + li];
  const int group = blockIdx.y;                    // 0 .. ngroups-1: full groups; ngroups: the narrow tail block
  const bool is_tail = group == a.ngroups;
  const int nblocks = a.ngroups + (a.tw > 0 ? 1 : 0);
  const int64_t slot_entries = (int64_t)a.ngroups * kGroupEntries + 256 * a.tw;
  const GH64* hist = a.hist_pool + (int64_t)a.gs.hist_slot[nid] * slot_entries + (int64_t)group * kGroupEntries;
  const int stride = is_tail ? a.tw : kSlots;      // accumulators per bin row
  const int slot = threadIdx.x & 31, seg = threadIdx.x >> 5;
  const int f = group * kSlots + slot;
  bool active = slot < stride && f < a.F && (a.feat_mask == nullptr || a.feat_mask[f] != 0);
  if (active && a.node_allowed != nullptr) active = a.node_allowed[(size_t)nid * a.F + f] != 0;
  if (a.feat_mask != nullptr && a.colsample_bynode < 1.0f) {
    // colsample_bynode: keep the max(1, floor(frac * |level set|)) features of the level's set with the smallest hash of this node
    __shared__ int s_rank[32], s_cnt;
    if (threadIdx.x < 32) s_rank[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const unsigned long long stream = 0x80000000ull + ((unsigned long long)(unsigned)*a.tree_index << 20) + (unsigned long long)nid;
    const float uf = rng_uniform(a.seed, stream, (unsigned long long)f);
    int rank = 0, cnt = 0;
    for (int g = seg; g < a.F; g += kEvalSegs) {
      if (a.feat_mask[g]) { ++cnt; const float ug = rng_uniform(a.seed, stream, (unsigned long long)g); rank += (ug < uf || (ug == uf && g < f)) ? 1 : 0; }
    }
    if (rank) atomicAdd(&s_rank[slot], rank);
    if (slot == 0 && cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    const int keep = max(1, (int)floorf(a.colsample_bynode * (float)s_cnt));
    active = active && s_rank[slot] < keep;
  }
  const int nbf = active ? a.cut_ptrs[f + 1] - a.cut_ptrs[f] : 0;
  const double isg = (double)a.gs.scales[2], ish = (double)a.gs.scales[3];
  const GH64 tot = a.gs.node_sum[nid];
  const double G = (double)tot.g * isg, H = (double)tot.h * ish;
  const bool mono = a.monotone != nullptr;
  const float w_lo = mono ? a.gs.lower[nid] : 0.f, w_hi = mono ? a.gs.upper[nid] : 0.f;
  const int mono_c = (mono && active) ? a.monotone[f] : 0;
  const float node_w = mono ? clamp_weight(calc_weight(a.p, G, H), w_lo, w_hi) : calc_weight(a.p, G, H);
  const float root_gain = mono ? gain_at_weight(a.p, G, H, node_w) : calc_gain(a.p, G, H);
  if (threadIdx.x == 0 && group == 0) { a.gs.root_gain[nid] = root_gain; a.gs.weight[nid] = node_w; }

  __shared__ long long segG[kEvalSegs][32], segH[kEvalSegs][32];
  __shared__ unsigned long long wkey[kEvalSegs];
  const int b0 = seg * kEvalBinsPerSeg;
  GH64 vals[kEvalBinsPerSeg];
  long long sG = 0, sH = 0;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerSeg; ++i) { int b = b0 + i; GH64 v; v.g = 0; v.h = 0; if (b < nbf) v = hist[b * stride + slot]; vals[i] = v; sG += v.g; sH += v.h; }
  segG[seg][slot] = sG; segH[seg][slot] = sH;
  __syncthreads();
  long long pG = 0, pH = 0, tG = 0, tH = 0;
#pragma unroll 8
  for (int s = 0; s < kEvalSegs; ++s) { long long x = segG[s][slot], y = segH[s][slot]; if (s < seg) { pG += x; pH += y; } tG += x; tH += y; }
  const bool fmiss = a.has_missing && (tG != tot.g || tH != tot.h);

  SplitCand best; best.loss_chg = 0.f; best.feature = 0; best.bin = -1; best.dleft = 0; best.ord = 0; best.GL = 0; best.HL = 0;
  unsigned long long bkey = 0ull;
  const double mcw = (double)a.p.min_child_weight;
  long long cG = pG, cH = pH;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerSeg; ++i) {          // forward scan: missing goes right, threshold = cut[b]
    int b = b0 + i;
    if (b < nbf) {
      GH64 v = vals[i]; cG += v.g; cH += v.h;
      double GL = (double)cG * isg, HL = (double)cH * ish;
      double GR = (double)(tot.g - cG) * isg, HR = (double)(tot.h - cH) * ish;
      if (HL >= mcw && HR >= mcw) {
        float lc;
        if (mono) { float gsum; lc = constrained_split_gain(a.p, GL, HL, GR, HR, w_lo, w_hi, mono_c, &gsum) ? gsum - root_gain : 0.0f; }
        else lc = calc_split_gain(a.p, GL, HL, GR, HR) - root_gain;
        unsigned long long k = cand_key(lc, f, b);
        if (k > bkey) { bkey = k; best.loss_chg = lc; best.feature = f; best.bin = b; best.dleft = 0; best.ord = b; best.GL = cG; best.HL = cH; }
      }
    }
  }
  if (fmiss) {                            // backward scan: missing goes left, threshold below bin b
    long long rG = tG - pG, rH = tH - pH;  // non-missing sum of bins >= b0
#pragma unroll
    for (int i = 0; i < kEvalBinsPerSeg; ++i) {
      int b = b0 + i;
      if (b < nbf) {
        long long lG = tot.g - rG, lH = tot.h - rH;       // left = everything else incl. missing
        double GL = (double)lG * isg, HL = (double)lH * ish, GR = (double)rG * isg, HR = (double)rH * ish;
        if (HR >= mcw && HL >= mcw) {
          float lc;
          if (mono) { float gsum; lc = constrained_split_gain(a.p, GL, HL, GR, HR, w_lo, w_hi, mono_c, &gsum) ? gsum - root_gain : 0.0f; }
          else lc = calc_split_gain(a.p, GL, HL, GR, HR) - root_gain;
          int ord = 256 + (255 - b);
          unsigned long long k = cand_key(lc, f, ord);
          if (k > bkey) { bkey = k; best.loss_chg = lc; best.feature = f; best.bin = b - 1; best.dleft = 1; best.ord = ord; best.GL = lG; best.HL = lH; }
        }
        GH64 v = vals[i]; rG -= v.g; rH -= v.h;
      }
    }
  }
  // block arg-max of the key
  unsigned long long k = bkey;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { unsigned long long x = __shfl_xor_sync(0xffffffffu, k, o); k = x > k ? x : k; }
  if ((threadIdx.x & 31) == 0) wkey[seg] = k;
  __syncthreads();
  unsigned long long m = 0ull;
#pragma unroll 8
  for (int s = 0; s < kEvalSegs; ++s) m = wkey[s] > m ? wkey[s] : m;
  SplitCand* out = a.gs.best_group + (size_t)nid * nblocks + group;
  if (m == 0ull) { if (threadIdx.x == 0) { SplitCand z; z.loss_chg = 0.f; z.feature = 0; z.bin = -1; z.dleft = 0; z.ord = 0; z.GL = 0; z.HL = 0; *out = z; } }
  else if (bkey == m) *out = best;        // keys are unique per (feature, ord)
}

// ---------------------------------------------------------------------------------------------
// block-wide exclusive scan over a global int array (single block), returns the total
// ---------------------------------------------------------------------------------------------
__device__ unsigned block_exclusive_scan(const unsigned* in, unsigned* out, int n, unsigned* s_tmp /*>=33*/) {
  unsigned carry = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int base = 0; base < n; base += blockDim.x) {
    int i = base + threadIdx.x;
    unsigned v = i < n ? in[i] : 0u, x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_tmp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned w = lane < nw ? s_tmp[lane] : 0u, z = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += y; }
      s_tmp[lane] = z - w;                       // exclusive warp offsets
      if (lane == 31) s_tmp[32] = z;             // chunk total
    }
    __syncthreads();
    if (i < n) out[i] = carry + s_tmp[warp] + x - v;
    carry += s_tmp[32];
    __syncthreads();
  }
  return carry;
}

// ---------------------------------------------------------------------------------------------
// node expansion, shared by the depth-wise (apply_kernel) and the loss-guided (apply_lossguide_kernel) policy
// ---------------------------------------------------------------------------------------------
// best split of nid over its candidate blocks (eval_kernel writes one per feature group and one for the tail); kept in gs.best
__device__ __forceinline__ SplitCand best_of_blocks(const ApplyArgs& a, int nid) {
  SplitCand best = a.gs.best_group[(size_t)nid * a.nblocks];
  unsigned long long bk = cand_key(best.loss_chg, best.feature, best.ord);
  for (int g = 1; g < a.nblocks; ++g) {
    SplitCand c = a.gs.best_group[(size_t)nid * a.nblocks + g];
    unsigned long long k = cand_key(c.loss_chg, c.feature, c.ord);
    if (k > bk) { bk = k; best = c; }
  }
  a.gs.best[nid] = best;
  return best;
}

// ExpandEntry::IsValid for a node at `depth` (max_leaves is the policy's: level order or queue order)
__device__ __forceinline__ bool split_is_valid(const TrainParamDev& p, const SplitCand& best, const GH64& tot, int depth) {
  bool ok = best.loss_chg > 1e-6f;
  if (ok && (best.HL == 0 || tot.h - best.HL == 0)) ok = false;
  if (ok && best.loss_chg < p.gamma) ok = false;
  if (ok && p.max_depth > 0 && depth >= p.max_depth) ok = false;
  return ok;
}

// the root was created without a parent: finish it once eval_kernel has its weight
__device__ __forceinline__ void finish_root(const ApplyArgs& a, double ish) {
  const GrowState& gs = a.gs; const TreeArrays& t = a.tree;
  t.base_weight[0] = gs.weight[0]; t.sum_hess[0] = (float)((double)gs.node_sum[0].h * ish); t.split_cond[0] = a.p.eta * gs.weight[0];
}

// Split nid by `best` into the new leaves Lc, Rc: tree arrays, the children's weight bounds and allowed features, their sums.
// Their row segments are set by part_kernel.
__device__ __forceinline__ void expand_node(const ApplyArgs& a, int nid, const SplitCand& best, const GH64& tot, int Lc, int Rc, double isg, double ish) {
  const GrowState& gs = a.gs; const TreeArrays& t = a.tree;
  const long long GLq = best.GL, HLq = best.HL, GRq = tot.g - best.GL, HRq = tot.h - best.HL;
  const double GL = (double)GLq * isg, HL = (double)HLq * ish, GR = (double)GRq * isg, HR = (double)HRq * ish;
  float wl = calc_weight(a.p, GL, HL), wr = calc_weight(a.p, GR, HR);
  if (a.monotone) {            // TreeEvaluator::AddSplit: children inherit the interval, mid bounds the constrained side
    const float lo = gs.lower[nid], hi = gs.upper[nid];
    wl = clamp_weight(wl, lo, hi); wr = clamp_weight(wr, lo, hi);
    const float mid = (wl + wr) / 2.0f; const int mc = a.monotone[best.feature];
    gs.lower[Lc] = lo; gs.upper[Lc] = hi; gs.lower[Rc] = lo; gs.upper[Rc] = hi;
    if (mc < 0) { gs.lower[Lc] = mid; gs.upper[Rc] = mid; } else if (mc > 0) { gs.upper[Lc] = mid; gs.lower[Rc] = mid; }
  }
  interaction_children(a, nid, best.feature, Lc, Rc);
  const int cb = a.cut_ptrs[best.feature];
  const float thr = best.dleft ? (best.bin < 0 ? a.min_vals[best.feature] : a.cut_vals[cb + best.bin]) : a.cut_vals[cb + best.bin];
  t.left[nid] = Lc; t.right[nid] = Rc; t.split_index[nid] = best.feature; t.split_cond[nid] = thr;
  t.split_bin[nid] = best.bin; t.default_left[nid] = (unsigned char)best.dleft;
  t.base_weight[nid] = gs.weight[nid]; t.loss_chg[nid] = best.loss_chg; t.sum_hess[nid] = (float)((double)tot.h * ish);
  const int ch[2] = {Lc, Rc}; const float cw[2] = {wl, wr}; const double chh[2] = {HL, HR};
  for (int s = 0; s < 2; ++s) {
    const int c = ch[s];
    t.left[c] = -1; t.right[c] = -1; t.parent[c] = nid; t.split_index[c] = 0; t.split_bin[c] = -1; t.default_left[c] = 0;
    t.split_cond[c] = a.p.eta * cw[s]; t.base_weight[c] = a.p.eta * cw[s]; t.loss_chg[c] = 0.f; t.sum_hess[c] = (float)chh[s];
  }
  gs.node_sum[Lc].g = GLq; gs.node_sum[Lc].h = HLq; gs.node_sum[Rc].g = GRq; gs.node_sum[Rc].h = HRq;
  gs.seg_begin[Lc] = 0; gs.seg_count[Lc] = 0; gs.seg_begin[Rc] = 0; gs.seg_count[Rc] = 0;
}

// Build list entry r for the children of nid: the child with the smaller hessian sum gets its histogram built into bld_slot,
// its sibling's (sub_slot) is the parent's minus it (subtract_kernel).
__device__ __forceinline__ void plan_child_hists(const GrowState& gs, int r, int nid, const SplitCand& best, const GH64& tot, int Lc, int Rc,
                                                 int bld_slot, int sub_slot) {
  const bool fewer_right = tot.h - best.HL < best.HL;
  const int bld = fewer_right ? Rc : Lc, sub = fewer_right ? Lc : Rc;
  gs.hist_slot[bld] = bld_slot; gs.hist_slot[sub] = sub_slot;
  gs.build_nid[r] = bld; gs.build_sub_nid[r] = sub; gs.build_parent_slot[r] = gs.hist_slot[nid];
}

// ---------------------------------------------------------------------------------------------
// depth-wise: expansion of one level (single block): the max_leaves order, child ids, level-region histogram slots, partition plan
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) apply_kernel(ApplyArgs a) {
  __shared__ unsigned s_tmp[33];
  GrowState& gs = a.gs;
  const int L = a.level;
  const int cnt = gs.level_count[L];
  const int* nodes = gs.level_nodes + (size_t)L * a.max_level_nodes;
  unsigned* valid = a.scratch;                       // [max_level_nodes]
  unsigned* rank = a.scratch + a.max_level_nodes;    // [max_level_nodes]
  unsigned* tiles = a.scratch + 2 * (size_t)a.max_level_nodes;
  const double isg = (double)gs.scales[2], ish = (double)gs.scales[3];
  if (L == 0 && threadIdx.x == 0 && cnt > 0) finish_root(a, ish);
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
    const int nid = nodes[i];
    const SplitCand best = best_of_blocks(a, nid);
    valid[i] = split_is_valid(a.p, best, gs.node_sum[nid], L) ? 1u : 0u;
  }
  __syncthreads();
  if (a.p.max_leaves > 0 && threadIdx.x == 0) {     // Driver::Pop order: increasing nid, stop at max_leaves
    int leaves = *gs.n_leaves;
    for (int i = 0; i < cnt; ++i) { if (valid[i]) { if (leaves >= a.p.max_leaves) valid[i] = 0; else ++leaves; } }
  }
  __syncthreads();
  const unsigned nvalid = block_exclusive_scan(valid, rank, cnt, s_tmp);
  const int n0 = *gs.n_nodes;
  const bool children_evaluated = (L + 1 < a.p.max_depth) || a.p.max_depth == 0;
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
    const int nid = nodes[i];
    tiles[i] = (gs.seg_count[nid] + kPartTile - 1) / kPartTile;
    gs.part_action[i] = (int)valid[i];
    if (!valid[i]) continue;
    const SplitCand best = gs.best[nid];
    const GH64 tot = gs.node_sum[nid];
    const int r = (int)rank[i];
    const int Lc = n0 + 2 * r, Rc = Lc + 1;
    expand_node(a, nid, best, tot, Lc, Rc, isg, ish);
    if (children_evaluated) {
      int* nxt = gs.level_nodes + (size_t)(L + 1) * a.max_level_nodes;
      nxt[2 * r] = Lc; nxt[2 * r + 1] = Rc;
      plan_child_hists(gs, r, nid, best, tot, Lc, Rc, a.next_base + r, a.next_base + a.next_half + r);
    }
  }
  __syncthreads();
  const unsigned total_tiles = block_exclusive_scan(tiles, gs.tile_prefix, cnt, s_tmp);
  if (threadIdx.x == 0) {
    gs.tile_prefix[cnt] = total_tiles;
    *gs.n_nodes = n0 + 2 * (int)nvalid;
    *gs.n_leaves += (int)nvalid;
    gs.level_count[L + 1] = children_evaluated ? 2 * (int)nvalid : 0;
    *gs.build_count = children_evaluated ? (int)nvalid : 0;
  }
}

// ---------------------------------------------------------------------------------------------
// grow_policy=lossguide: one node per iteration (upstream Driver::Pop in loss-guided mode: the open candidate with the largest
// loss_chg, ties to the smaller node id; an INVALID top candidate ends the tree).  Node expansion is shared with apply_kernel,
// with "level" 0 = the node being split and "level" 1 = its two children: this kernel (a) registers the candidates evaluated by
// the previous iteration, (b) picks and validates the best one, (c) expands it.
// Histogram slots: the built child gets a fresh slot, its sibling inherits the parent's (subtract_kernel works in place).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) apply_lossguide_kernel(ApplyArgs a, int iter) {
  __shared__ unsigned long long s_key[8];
  GrowState& gs = a.gs;
  const double isg = (double)gs.scales[2], ish = (double)gs.scales[3];
  const int src = iter == 0 ? 0 : 1;
  const int cnt = gs.level_count[src];
  const int* nodes = gs.level_nodes + (size_t)src * a.max_level_nodes;
  if (iter == 0 && threadIdx.x == 0 && cnt > 0) finish_root(a, ish);
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) {        // (a) Driver::Push: candidates with loss_chg > eps enter the queue
    const int nid = nodes[i];
    gs.open[nid] = best_of_blocks(a, nid).loss_chg > 1e-6f ? 1 : 0;
  }
  __syncthreads();
  const int n0 = *gs.n_nodes;
  unsigned long long key = 0ull;                               // (b) arg-max of (loss_chg, -nid) over the open candidates
  for (int nid = threadIdx.x; nid < n0; nid += blockDim.x)
    if (gs.open[nid]) { unsigned long long k = ((unsigned long long)__float_as_uint(gs.best[nid].loss_chg) << 32) | (unsigned long long)(0xffffffffu - (unsigned)nid); key = k > key ? k : key; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { unsigned long long x = __shfl_xor_sync(0xffffffffu, key, o); key = x > key ? x : key; }
  if ((threadIdx.x & 31) == 0) s_key[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < 8; ++w) key = s_key[w] > key ? s_key[w] : key;
  bool stop = *gs.lg_done != 0 || key == 0ull;
  int nid = 0; SplitCand best{}; GH64 tot{};
  if (!stop) {
    nid = (int)(0xffffffffu - (unsigned)(key & 0xffffffffull));
    best = gs.best[nid]; tot = gs.node_sum[nid];
    stop = !split_is_valid(a.p, best, tot, gs.depth[nid]) || (a.p.max_leaves > 0 && *gs.n_leaves == a.p.max_leaves);
  }
  if (stop) {
    *gs.lg_done = 1;
    gs.level_count[0] = 0; gs.level_count[1] = 0; *gs.build_count = 0; gs.part_action[0] = 0; gs.tile_prefix[0] = 0; gs.tile_prefix[1] = 0;
    return;
  }
  gs.open[nid] = 0;                                            // (c) expand
  const int Lc = n0, Rc = n0 + 1, d = gs.depth[nid];
  expand_node(a, nid, best, tot, Lc, Rc, isg, ish);
  gs.depth[Lc] = d + 1; gs.depth[Rc] = d + 1; gs.open[Lc] = 0; gs.open[Rc] = 0;
  *gs.n_nodes = n0 + 2;
  const int leaves = *gs.n_leaves + 1;
  *gs.n_leaves = leaves;
  // ExpandEntry::ChildIsValid: children that could never split are not evaluated (no partition, no histogram)
  const bool children_evaluated = !(a.p.max_depth > 0 && d + 1 >= a.p.max_depth) && !(a.p.max_leaves > 0 && leaves >= a.p.max_leaves);
  gs.level_nodes[0] = nid; gs.level_count[0] = 1;
  gs.part_action[0] = children_evaluated ? 1 : 0;
  gs.tile_prefix[0] = 0; gs.tile_prefix[1] = children_evaluated ? (gs.seg_count[nid] + kPartTile - 1) / kPartTile : 0u;
  if (children_evaluated) {
    int* nxt = gs.level_nodes + (size_t)a.max_level_nodes;
    nxt[0] = Lc; nxt[1] = Rc; gs.level_count[1] = 2;
    const int slot = (*gs.n_slots)++;
    plan_child_hists(gs, 0, nid, best, tot, Lc, Rc, slot, gs.hist_slot[nid]);
    *gs.build_count = 1;
  } else { gs.level_count[1] = 0; *gs.build_count = 0; }
}

// lossguide keeps every live row segment in ONE buffer set: the children written by the partition go straight back
template <typename Pay>       // the partition's payload: float2 (g,h) or float g
__global__ void __launch_bounds__(256) lg_copy_back_kernel(PartArgs a, unsigned* ridx_dst, Pay* gp_dst, unsigned* tl_dst) {
  const GrowState& gs = a.gs;
  if (gs.level_count[0] <= 0 || !gs.part_action[0]) return;
  const int nid = gs.level_nodes[0];
  const unsigned b = gs.seg_begin[nid], c = gs.seg_count[nid];
  const Pay* gp_src = static_cast<const Pay*>(a.gp_next);
  for (unsigned p = b + blockIdx.x * blockDim.x + threadIdx.x; p < b + c; p += gridDim.x * blockDim.x) {
    ridx_dst[p] = a.ridx_next[p]; gp_dst[p] = gp_src[p];
    if (a.tl_next) tl_dst[p] = a.tl_next[p];
  }
}

__global__ void __launch_bounds__(256) zero_build_slots_kernel(GrowState gs, GH64* pool, size_t stride) {
  const int r = blockIdx.x;
  if (r >= *gs.build_count) return;
  GH64* h = pool + (size_t)gs.hist_slot[gs.build_nid[r]] * stride;
  GH64 z; z.g = 0; z.h = 0;
  for (size_t e = (size_t)blockIdx.y * blockDim.x + threadIdx.x; e < stride; e += (size_t)gridDim.y * blockDim.x) h[e] = z;
}

// multi-rank lossguide: the collective needs a fixed address, the freshly built slot is chosen on the device
__global__ void __launch_bounds__(256) lg_stage_kernel(GrowState gs, GH64* pool, size_t stride, int to_stage) {
  if (*gs.build_count <= 0) return;
  GH64* slot = pool + (size_t)gs.hist_slot[gs.build_nid[0]] * stride;
  GH64* stage = pool + (size_t)kLgStageSlot * stride;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < stride; e += (size_t)gridDim.x * blockDim.x) {
    if (to_stage) stage[e] = slot[e]; else slot[e] = stage[e];
  }
}

// ---------------------------------------------------------------------------------------------
// row partition: one pass per level.  A tile is kPartTile consecutive positions of one node's segment.  Lefts fill the
// children's segment from its start and rights from its end downward, so a tile only needs the lefts of the node's EARLIER
// tiles (decoupled look-back), never the node's left total: a right child holds its rows in reverse parent order, which no
// consumer depends on (histogram sums are exact integers).  Rows of nodes that stay leaves drop out of the row-id buffer.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int find_node_of_tile(const unsigned* tile_prefix, int cnt, unsigned tile) {
  int lo = 0, hi = cnt;        // largest i with tile_prefix[i] <= tile
  while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (tile_prefix[mid] <= tile) lo = mid; else hi = mid; }
  return lo;
}

// Look-back descriptor of a tile: status in the top two bits, a row count in the low 32.
constexpr unsigned long long kDescAggregate = 1ull << 62;   // the tile's own left count
constexpr unsigned long long kDescPrefix = 2ull << 62;      // lefts of the node's tiles up to and including this one

__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// one warp: lefts of the tiles d[0 .. lt-1], read 32 descriptors at a time from the nearest down to the first PREFIX.
// Every tile waited for belongs to a CTA that took its ticket earlier (so it is running) and publishes its aggregate
// before it waits for anything.
__device__ unsigned lookback_lefts(const unsigned long long* d, unsigned lt) {
  const int lane = threadIdx.x & 31;
  unsigned acc = 0;
  for (int hi = (int)lt - 1; hi >= 0; hi -= 32) {
    const int j = hi - lane;
    unsigned long long v = 0;
    if (j >= 0) { v = ld_relaxed_u64(d + j); while ((v >> 62) == 0) { __nanosleep(64); v = ld_relaxed_u64(d + j); } }
    const unsigned pref = __ballot_sync(0xffffffffu, (v >> 62) == 2);
    const int last = pref ? __ffs(pref) - 1 : 31;         // nearest tile that carries a prefix ends the sum
    unsigned x = lane <= last ? (unsigned)v : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    acc += x;
    if (pref) break;
  }
  return acc;
}

// One CTA per tile, taken from an atomic ticket.  Per tile: ids, payload and the split byte in; the left count published; the
// tile compacted in shared memory ([lefts | rights], position order) while warp 0 looks back; id + payload per row out.
// The node's last tile writes the children's segments; the last CTA of the grid computes the build list's prefix.
// Payload: GONLY (constant hessian) carries g alone, else (g,h); TL adds the row's 4 tail bytes.  8, 12 or 16 B per row out.
// The tile is latency bound (a dependent split-byte gather per row): the G-only variants fit 6 / 5 CTAs per SM in 40 / 48
// registers without spilling, and each CTA more per SM measured faster; the (g,h) variants keep 4 (64 registers).
template <bool GONLY, bool TL>
__global__ void __launch_bounds__(256, GONLY ? (TL ? 5 : 6) : 4) part_kernel(PartArgs a) {
  typedef typename std::conditional<GONLY, float, float2>::type Pay;
  GrowState& gs = a.gs;
  __shared__ unsigned s_rid[kPartTile];
  __shared__ Pay s_gp[kPartTile];
  __shared__ unsigned s_tl[TL ? kPartTile : 1];
  __shared__ unsigned s_w[8];
  const int cnt = gs.level_count[a.level];
  const unsigned total = cnt > 0 ? gs.tile_prefix[cnt] : 0u;
  if (threadIdx.x == 0) s_w[0] = atomicAdd(gs.part_ctl, 1u);
  __syncthreads();
  const unsigned tile = s_w[0];
  __syncthreads();
  const int i = tile < total ? find_node_of_tile(gs.tile_prefix, cnt, tile) : 0;
  if (tile < total && gs.part_action[i]) {
    const int nid = gs.level_nodes[(size_t)a.level * a.max_level_nodes + i];
    const unsigned t0 = gs.tile_prefix[i], lt = tile - t0;
    const unsigned b = gs.seg_begin[nid], c = gs.seg_count[nid];
    const unsigned p0 = b + lt * kPartTile, p1 = (b + c < p0 + kPartTile) ? b + c : p0 + kPartTile;
    const unsigned nrows = p1 - p0;
    const int f = a.tree.split_index[nid];
    const int sb = a.tree.split_bin[nid], dl = a.tree.default_left[nid];
    const uint8_t* col = a.bins_col + (int64_t)f * a.n;        // column-major copy: one byte per row
    const Pay* gp_cur = static_cast<const Pay*>(a.gp_cur);
    Pay* gp_next = static_cast<Pay*>(a.gp_next);
    const unsigned pt = p0 + threadIdx.x * 8;
    unsigned rows[8]; Pay gp[8]; unsigned tl[8]; unsigned char fl[8]; unsigned mine = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const unsigned p = pt + j;
      rows[j] = 0; gp[j] = Pay{}; tl[j] = 0u;
      if (p < p1) {
        rows[j] = a.ridx_cur ? a.ridx_cur[p] : p;
        if constexpr (GONLY) gp[j] = static_cast<const float*>(a.gp_cur)[(size_t)p * a.gp_cur_stride];
        else gp[j] = gp_cur[p];
        if constexpr (TL) tl[j] = a.tl_cur[p];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (pt + j < p1) {
        const int byte = col[rows[j]];
        const bool left = (a.has_missing && byte == kMissingBin) ? (dl != 0) : (byte <= sb);
        fl[j] = left ? 1 : 0; mine += fl[j];
      } else fl[j] = 2;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned x = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { unsigned y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    unsigned woff = 0, tile_left = 0;
    for (int w = 0; w < 8; ++w) { if (w < warp) woff += s_w[w]; tile_left += s_w[w]; }
    unsigned long long* desc = gs.tile_desc + t0;
    if (threadIdx.x == 0) st_relaxed_u64(desc + lt, (lt == 0 ? kDescPrefix : kDescAggregate) | tile_left);
    unsigned lbefore = woff + x - mine;               // lefts before my first position inside the tile
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (fl[j] == 2) continue;
      const unsigned jj = threadIdx.x * 8 + j;
      const unsigned slot = fl[j] ? lbefore++ : tile_left + (jj - lbefore);
      s_rid[slot] = rows[j]; s_gp[slot] = gp[j]; if constexpr (TL) s_tl[slot] = tl[j];
    }
    unsigned lefts_before = 0;
    if (warp == 0 && lt > 0) {
      lefts_before = lookback_lefts(desc, lt);
      if (lane == 0) st_relaxed_u64(desc + lt, kDescPrefix | (lefts_before + tile_left));
    }
    __syncthreads();                                  // every thread has read the warp totals: s_w[0] is free
    if (threadIdx.x == 0) s_w[0] = lefts_before;
    __syncthreads();
    lefts_before = s_w[0];
    const unsigned rights_before = lt * kPartTile - lefts_before;
    const int Lc = a.tree.left[nid], Rc = a.tree.right[nid];
    bool write_left = true, write_right = true;
    if (a.build_only) { const bool build_right = gs.node_sum[Rc].h < gs.node_sum[Lc].h; write_left = !build_right; write_right = build_right; }
    const unsigned k0 = write_left ? 0u : tile_left, k1 = write_right ? nrows : tile_left;
    // lefts to b + lefts_before + k, rights to b + c - 1 - (rights_before + k): two contiguous, coalesced streams
    const unsigned dl0 = b + lefts_before, dr0 = b + c - 1 - rights_before + tile_left;
    for (unsigned k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
      const unsigned dest = k < tile_left ? dl0 + k : dr0 - k;
      a.ridx_next[dest] = s_rid[k];
      gp_next[dest] = s_gp[k];
      if constexpr (TL) a.tl_next[dest] = s_tl[k];
    }
    if (threadIdx.x == 0) {
      if (lt == gs.tile_prefix[i + 1] - t0 - 1) {       // the node's last tile knows its left total
        const unsigned nl = lefts_before + tile_left;
        gs.seg_begin[Lc] = b; gs.seg_count[Lc] = nl; gs.seg_begin[Rc] = b + nl; gs.seg_count[Rc] = c - nl;
      }
      if (a.rows_counter) { atomicAdd(a.rows_counter, (unsigned long long)nrows); atomicAdd(a.rows_counter + 1, (unsigned long long)(k1 - k0)); }
    }
  }
  // the last CTA to finish sees every child segment: exclusive prefix of the build list's row counts (+ total)
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); s_w[0] = atomicAdd(gs.part_ctl + 1, 1u) == gridDim.x - 1 ? 1u : 0u; }
  __syncthreads();
  if (!s_w[0]) return;
  __threadfence();
  const int nb = *gs.build_count;
  for (int r = threadIdx.x; r < nb; r += blockDim.x) gs.build_prefix[r] = __ldcg(gs.seg_count + gs.build_nid[r]);
  __syncthreads();
  const unsigned tot = nb > 0 ? block_exclusive_scan(gs.build_prefix, gs.build_prefix, nb, s_rid /* >= 33 words, free now */) : 0u;
  if (threadIdx.x == 0) gs.build_prefix[nb > 0 ? nb : 0] = tot;
}

// Prediction-cache update of a finished tree: one streaming pass in ROW order over the column-major bins
// (coalesced, no scattered read-modify-write of the cache).  The tree is packed into shared memory first
// (8 B per node) so that a traversal step costs one LDS + one global byte load.  The feature id keeps all its bits; the right
// child is left + 1 (both growth policies allocate the children as an adjacent pair).
struct PackedNode { unsigned feat; unsigned short bin_dl; unsigned short left; };   // bin_dl: (split_bin + 1) | dl << 15; left == 0xffff: leaf
constexpr int kPackedNodesSmem = 2048;
static_assert(sizeof(PackedNode) == 8, "PackedNode is 8 B");

__global__ void __launch_bounds__(256) update_margin_kernel(TreeArrays t, const int* n_nodes, const uint8_t* bins_col, int64_t n, int has_missing,
                                                            float* margin, int K, int k) {
  __shared__ PackedNode s_nodes[kPackedNodesSmem];
  __shared__ float s_leaf[kPackedNodesSmem];
  const int nn = *n_nodes;
  const bool packed = nn <= kPackedNodesSmem && nn < 0xffff;
  if (packed) {
    for (int i = threadIdx.x; i < nn; i += blockDim.x) {
      PackedNode p; p.feat = (unsigned)t.split_index[i]; p.bin_dl = (unsigned short)((t.split_bin[i] + 1) | (t.default_left[i] ? 0x8000 : 0));
      const int l = t.left[i]; p.left = l < 0 ? 0xffff : (unsigned short)l;
      s_nodes[i] = p; s_leaf[i] = t.split_cond[i];
    }
    __syncthreads();
  }
  // four independent traversals per thread (rows r, r+256, r+512, r+768 of the block's 1024-row tile): 4 loads in flight
  const int64_t base = (int64_t)blockIdx.x * 1024 + threadIdx.x;
  int nid[4]; bool done[4];
  const bool root_leaf = packed ? (s_nodes[0].left == 0xffff) : (t.left[0] == -1);
#pragma unroll
  for (int j = 0; j < 4; ++j) { nid[j] = 0; done[j] = (base + j * 256 >= n) || root_leaf; }
  bool any = !(done[0] && done[1] && done[2] && done[3]);
  while (any) {
    int byte[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int f = packed ? (int)s_nodes[nid[j]].feat : t.split_index[nid[j]];
      byte[j] = done[j] ? 0 : bins_col[(int64_t)f * n + base + j * 256];
    }
    any = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (done[j]) continue;
      const int nd = nid[j];
      if (packed) {
        const PackedNode p = s_nodes[nd];
        const bool left = (has_missing && byte[j] == kMissingBin) ? ((p.bin_dl & 0x8000) != 0) : (byte[j] < (int)(p.bin_dl & 0x7fff));
        nid[j] = left ? p.left : p.left + 1;
        done[j] = s_nodes[nid[j]].left == 0xffff;
      } else {
        const bool left = (has_missing && byte[j] == kMissingBin) ? (t.default_left[nd] != 0) : (byte[j] <= t.split_bin[nd]);
        nid[j] = left ? t.left[nd] : t.right[nd];
        done[j] = t.left[nid[j]] == -1;
      }
      any |= !done[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { const int64_t r = base + j * 256; if (r < n) margin[r * K + k] += packed ? s_leaf[nid[j]] : t.split_cond[nid[j]]; }
}

// sibling = parent - built child (exact int64)
__global__ void __launch_bounds__(256) subtract_kernel(GrowState gs, GH64* pool, size_t stride) {
  const int r = blockIdx.x;
  if (r >= *gs.build_count) return;
  const int bld = gs.build_nid[r], sub = gs.build_sub_nid[r];
  const GH64* hb = pool + (size_t)gs.hist_slot[bld] * stride;
  const GH64* hp = pool + (size_t)gs.build_parent_slot[r] * stride;
  GH64* hs = pool + (size_t)gs.hist_slot[sub] * stride;
  for (size_t e = (size_t)blockIdx.y * blockDim.x + threadIdx.x; e < stride; e += (size_t)gridDim.y * blockDim.x) {
    GH64 p = hp[e], b = hb[e]; GH64 o; o.g = p.g - b.g; o.h = p.h - b.h; hs[e] = o;
  }
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
void launch_init_tree(const GrowState& gs, const TreeArrays& t, unsigned n, cudaStream_t s) {
  init_tree_kernel<<<1, 32, 0, s>>>(gs, t, n); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_scales(const GrowState& gs, int grad_bits, cudaStream_t s) { scales_kernel<<<1, 32, 0, s>>>(gs, grad_bits); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
void launch_eval(const EvalArgs& a, int max_nodes_level, cudaStream_t s) {
  dim3 grid(max_nodes_level, a.ngroups + (a.tw > 0 ? 1 : 0)); eval_kernel<<<grid, 32 * kEvalSegs, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_apply_lossguide(const ApplyArgs& a, int iter, cudaStream_t s) { apply_lossguide_kernel<<<1, 256, 0, s>>>(a, iter); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
void launch_lg_copy_back(const PartArgs& a, unsigned* ridx_dst, void* gp_dst, unsigned* tl_dst, unsigned max_tiles, cudaStream_t s) {
  const unsigned grid = max_tiles < 1184u ? max_tiles : 1184u;
  if (a.g_only) lg_copy_back_kernel<float><<<grid, 256, 0, s>>>(a, ridx_dst, static_cast<float*>(gp_dst), tl_dst);
  else lg_copy_back_kernel<float2><<<grid, 256, 0, s>>>(a, ridx_dst, static_cast<float2*>(gp_dst), tl_dst);
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_zero_build_slots(const GrowState& gs, GH64* pool, size_t slot_entries, int max_build, cudaStream_t s) {
  dim3 grid(max_build, (unsigned)((slot_entries + 1023) / 1024)); zero_build_slots_kernel<<<grid, 256, 0, s>>>(gs, pool, slot_entries); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_lg_stage(const GrowState& gs, GH64* pool, size_t slot_entries, int to_stage, cudaStream_t s) {
  lg_stage_kernel<<<(unsigned)((slot_entries + 1023) / 1024), 256, 0, s>>>(gs, pool, slot_entries, to_stage); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_apply(const ApplyArgs& a, cudaStream_t s) { apply_kernel<<<1, 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError()); }
void launch_partition(const PartArgs& a, unsigned max_tiles, cudaStream_t s) {
  CUDA_OK(cudaMemsetAsync(a.gs.tile_desc, 0, sizeof(unsigned long long) * ((size_t)max_tiles + 1), s));   // descriptors + part_ctl
  const bool tl = a.tl_cur != nullptr;
  if (a.g_only) { if (tl) part_kernel<true, true><<<max_tiles, 256, 0, s>>>(a); else part_kernel<true, false><<<max_tiles, 256, 0, s>>>(a); }
  else { if (tl) part_kernel<false, true><<<max_tiles, 256, 0, s>>>(a); else part_kernel<false, false><<<max_tiles, 256, 0, s>>>(a); }
  ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_update_margin(const TreeArrays& t, const int* n_nodes, const uint8_t* bins_col, int64_t n, int has_missing, float* margin, int K, int k, cudaStream_t s) {
  if (n == 0) return;
  update_margin_kernel<<<(unsigned)((n + 1023) / 1024), 256, 0, s>>>(t, n_nodes, bins_col, n, has_missing, margin, K, k); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}
void launch_subtract(const GrowState& gs, GH64* pool, size_t slot_entries, int max_build, cudaStream_t s) {
  dim3 grid(max_build, (unsigned)((slot_entries + 1023) / 1024)); subtract_kernel<<<grid, 256, 0, s>>>(gs, pool, slot_entries); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
