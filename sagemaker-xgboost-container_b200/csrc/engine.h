// engine.h -- internal declarations shared by the CUDA translation units of libb200xgb.so.
// Product code: H100 (sm_90a) gradient-boosted-tree trainer/predictor behind the xgboost C API
// surface that the SageMaker XGBoost container reaches through `import xgboost` (SURVEY.md section 8b).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200 {

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
struct Error : std::runtime_error { using std::runtime_error::runtime_error; };
#define B200_CHECK(cond, msg) do { if (!(cond)) throw ::b200::Error(std::string(msg)); } while (0)
#define CUDA_OK(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) throw ::b200::Error( \
    std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); } while (0)

// number of kernels this library has launched (reported by bench.py as gpu_launches)
extern long long g_kernel_launches;

// the engine's stream, and the streaming multiprocessors of its device (grid sizes of the grid-stride kernels scale with it)
cudaStream_t engine_stream();
int engine_num_sms();

// bytes held through DevBuf, now and at most since the last reset (include/b200xgb.h XGB200DeviceMemory)
void devmem_note(int64_t delta);
void devmem_query(uint64_t* live, uint64_t* peak, bool reset_peak);

template <typename T> struct DevBuf {
  T* p = nullptr; size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() { if (p) { cudaFree(p); devmem_note(-(int64_t)(n * sizeof(T))); } p = nullptr; n = 0; }
  void alloc(size_t count) { if (count == n && p) return; release();
    if (count) { CUDA_OK(cudaMalloc(&p, count * sizeof(T))); devmem_note((int64_t)(count * sizeof(T))); } n = count; }
  void ensure(size_t count) { if (count > n) alloc(count); }
  void zero(cudaStream_t s) { if (n) CUDA_OK(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
};

// ---------------------------------------------------------------------------------------------
// layout constants (DESIGN.md "data layout in HBM")
// ---------------------------------------------------------------------------------------------
constexpr int kSlots = 32;            // feature slots per group == bytes per row slice == one 32 B sector
constexpr int kBins = 256;            // bins per feature (uint8 codes); code 255 = missing when has_missing
constexpr int kGroupEntries = kBins * kSlots;          // (bin, slot) accumulators per feature group
constexpr int kMissingBin = 255;
// Fixed-point grid of the gradients: |g_q| <= 2^bits, h_q <= 2^(bits+1), and a CTA checks its int32 accumulators for overflow
// every `window` rows with window * 2^bits = 2^31 - 2^25 (hist.cu kSpillThresholdG / H: what may stay between windows).  Large matrices use 18 bits / 8064 rows; matrices up to 2^20 rows
// (where one-row leaves with large gradients are common and the extra overflow checks cost nothing measurable) use
// 21 bits / 1008 rows, which keeps even a single-row leaf within 1e-5 of the double-precision reference.
constexpr int kGradBits = 18, kWindowRows = 8064;
constexpr int kGradBitsSmall = 21, kWindowRowsSmall = 1008;
constexpr int64_t kSmallMatrixRows = 1 << 20;
inline int grad_bits_for(int64_t n) { return n <= kSmallMatrixRows ? kGradBitsSmall : kGradBits; }
inline int window_rows_for(int64_t n) { return n <= kSmallMatrixRows ? kWindowRowsSmall : kWindowRows; }
constexpr int kMaxDepth = 16;
// Widest training matrix: eval_kernel runs one block row per feature group (+ the tail block) in grid.y (<= 65535), and the
// split key (tree.cu cand_key) holds 23 bits of feature id.
constexpr int kMaxTrainFeatures = 65534 * 32;
static_assert(kMaxTrainFeatures < (1 << 23), "cand_key holds 23 bits of feature id");

struct GH64 { long long g, h; };      // exact fixed-point gradient/hessian sums

// Binned matrix (DESIGN.md "data layout in HBM"): features are laid out in full 32-wide groups plus an optional narrow
// tail so that neither HBM traffic nor shared-memory atomics are spent on pad slots (F = 100 -> 3 groups + a 4-wide tail):
//   main  row-major [n][ngroups*32 B]   feature f < ngroups*32 -> group f >> 5, slot f & 31
//   tail  row-major [n][tw B]           feature f >= ngroups*32 -> tail slot f - ngroups*32   (tw in {0, 4, 8})
// plus a column-major copy [F][n] for the one-byte-per-row consumers (partition, prediction-cache update).
struct BinnedMatrix {
  const uint8_t* bins = nullptr;
  const uint8_t* bins_tail = nullptr;
  const uint8_t* bins_col = nullptr;
  const uint8_t* bins_gather = nullptr;   // main block with rows padded to whole 128 B lines when ngroups * 32 == 96 (else == bins)
  int gather_stride = 0;                  // DRAM serves gathered rows in whole 128 B lines: an aligned 96 B row costs one, a packed one 1.5
  int tail_in_gather = 0;                 // the aligned copy also holds each row's 8 tail bytes (tw == 8), at offset ngroups * 32 (in the pad)
  int64_t n = 0;
  int F = 0, ngroups = 0, tw = 0, ntail = 0;
  int has_missing = 0;
  int unused = 0;                         // makes the padding explicit: grow.h TreeInputs compares this block as bytes
};

// F = 32 a + L: a tail exists when there is at least one full group and 1 <= L <= 8; otherwise L features get a padded group.
inline void feature_layout(int F, int* ngroups, int* tw, int* ntail) {
  const int a = F / 32, L = F % 32;
  if (a >= 1 && L >= 1 && L <= 8) { *ngroups = a; *ntail = L; *tw = L <= 4 ? 4 : 8; }
  else { *ngroups = a + (L > 0 ? 1 : 0); if (*ngroups == 0) *ngroups = 1; *ntail = 0; *tw = 0; }
}
// (g,h) accumulators of one histogram-pool slot: [ngroups][256][32] then the tail [256][tw]
inline size_t hist_slot_entries(int ngroups, int tw) { return (size_t)ngroups * 256 * 32 + (size_t)256 * tw; }

// ---------------------------------------------------------------------------------------------
// training parameters (names follow the container's hyperparameter schema,
// reference: src/sagemaker_xgboost_container/algorithm_mode/hyperparameter_validation.py:141-346)
// ---------------------------------------------------------------------------------------------
enum Objective : int { kSquaredError = 0, kBinaryLogistic = 1, kRegLogistic = 2, kLogitRaw = 3, kSoftprob = 4, kSoftmax = 5,
                       kSquaredLogError = 6, kPseudoHuber = 7, kPoisson = 8, kGamma = 9, kTweedie = 10, kHinge = 11,
                       kAft = 12, kCox = 13,         // survival objectives: own gradient kernels (survival.cu), not gradient_kernel
                       kAbsoluteError = 14,          // own gradient kernel and a leaf refresh after every tree (adaptive.cu)
                       kQuantileError = 15,          // likewise, one output (and one tree per round) per quantile_alpha
                       kRankPairwise = 16, kRankNdcg = 17, kRankMap = 18 };   // over query groups: own gradient kernels (rank.cu)
// prediction transform of an objective (upstream ObjFunction::PredTransform / ProbToMargin): 0 identity, 1 sigmoid / logit,
// 2 exp / log (count:poisson, reg:gamma, reg:tweedie, survival:aft, survival:cox), 3 step at 0 (binary:hinge; its margin is the raw score)
enum Transform : int { kTransformNone = 0, kTransformSigmoid = 1, kTransformExp = 2, kTransformHinge = 3 };
inline bool objective_is_logistic(int o) { return o == kBinaryLogistic || o == kRegLogistic || o == kLogitRaw; }
inline bool objective_is_log_link(int o) { return o == kPoisson || o == kGamma || o == kTweedie; }
inline bool objective_is_survival(int o) { return o == kAft || o == kCox; }
// the objective sets each leaf of a grown tree to a quantile of its rows' residuals (upstream ObjFunction::Task().UpdateTreeLeaf())
inline bool objective_is_adaptive(int o) { return o == kAbsoluteError || o == kQuantileError; }
inline bool objective_is_rank(int o) { return o == kRankPairwise || o == kRankNdcg || o == kRankMap; }
inline int objective_transform(int o) {
  if (o == kBinaryLogistic || o == kRegLogistic) return kTransformSigmoid;
  if (objective_is_log_link(o) || objective_is_survival(o)) return kTransformExp;
  return o == kHinge ? kTransformHinge : kTransformNone;
}

struct TrainParam {
  int objective = kSquaredError;
  int num_class = 1;
  int max_depth = 6, max_leaves = 0, max_bin = 256;
  int lossguide = 0;            // grow_policy: 0 depthwise, 1 lossguide
  float eta = 0.3f, lambda = 1.0f, alpha = 0.0f, gamma = 0.0f, min_child_weight = 1.0f, max_delta_step = 0.0f;
  float scale_pos_weight = 1.0f, subsample = 1.0f, colsample_bytree = 1.0f, colsample_bylevel = 1.0f, colsample_bynode = 1.0f;
  unsigned seed = 0;
  int num_parallel_tree = 1;    // trees per class per boosting round (boosted random forests)
  int gradient_based = 0;       // sampling_method: 0 uniform, 1 gradient_based (sampling.h; only with subsample < 1)
  float huber_slope = 1.0f, tweedie_variance_power = 1.5f, poisson_max_delta_step = 0.7f;   // objective parameters (upstream defaults)
  int aft_dist = 0; float aft_sigma = 1.0f;     // survival:aft: aft_loss_distribution (survival.h AftDist), aft_loss_distribution_scale
  std::vector<float> quantile_alpha;            // reg:quantileerror: one output per entry (empty for every other objective)
  // rank:* (upstream LambdaRankParam): lambdarank_num_pair_per_sample (the topk truncation K), ndcg_exp_gain,
  // lambdarank_normalization, lambdarank_score_normalization, lambdarank_bias_norm (inert: lambdarank_unbiased is rejected)
  // lambdarank_unbiased=true is read and written, and a model with it predicts, but it does not train
  int rank_mean = 0, rank_unbiased = 0, rank_k = 32, rank_exp_gain = 1, rank_normalization = 1, rank_score_normalization = 1; float rank_bias_norm = 2.0f;
  // Outputs per row: margin columns, trees per round and layer (times num_parallel_tree), prediction columns.  num_class
  // itself is the class count of multi:* (softmax, merror / mlogloss) and 1 otherwise.
  int num_outputs() const { return objective == kQuantileError ? (int)quantile_alpha.size() : num_class; }
};

// ---------------------------------------------------------------------------------------------
// device-side tree-growing state (one per Booster; all control decisions stay on the device so a
// whole tree is one stream of launches with no host synchronisation)
// ---------------------------------------------------------------------------------------------
struct SplitCand {
  float loss_chg; int feature; int bin; int dleft; int ord;
  long long GL, HL;                   // fixed-point left sums (right = node - left)
};

struct TreeArrays {                   // capacity max_nodes each; the layout the model file stores
  int *left, *right, *parent, *split_index, *split_bin;
  unsigned char* default_left;
  float *split_cond, *base_weight, *loss_chg, *sum_hess;
};

struct GrowState {
  // per tree-node (indexed by nid)
  unsigned* seg_begin; unsigned* seg_count;     // row segment in the row-index buffer
  int* hist_slot;                               // slot in the histogram pool
  GH64* node_sum;                               // exact node totals
  float* root_gain; float* weight;
  SplitCand* best;                              // reduced over groups
  SplitCand* best_group;                        // [nid][ngroups + (tail ? 1 : 0)]
  // per level
  int* level_nodes;                             // [kMaxDepth+1][max_level_nodes] nids alive at each depth
  int* level_count;                             // [kMaxDepth+2]
  // build list of the level being built
  int* build_nid; int* build_sub_nid; int* build_parent_slot; int* build_count;   // build_count[0]
  unsigned* build_prefix;                       // exclusive prefix of seg_count over the build list (+ total)
  // partition plan of the level being split
  int* part_action;                             // per alive node index at level: 0 leaf, 1 split
  unsigned* tile_prefix;                        // per alive node: exclusive prefix of tile counts (+ total)
  unsigned long long* tile_desc;                // per tile: look-back descriptor (status | left count or inclusive prefix)
  unsigned* part_ctl;                           // [0] tile ticket, [1] finished CTAs; zeroed with tile_desc before every partition
  int* n_nodes; int* n_leaves;
  // grow_policy=lossguide: depth and open-candidate flag per node, next free histogram slot, sticky end-of-tree flag
  int* depth; unsigned char* open; int* n_slots; int* lg_done;
  // monotone constraints: weight bounds per node (upstream TreeEvaluator lower_bounds_ / upper_bounds_)
  float* lower; float* upper;
  float* scales;                                // [0]=sg [1]=sh [2]=1/sg [3]=1/sh
  unsigned* absmax;                             // [0]=max|g| bits [1]=max h bits
};

}  // namespace b200
