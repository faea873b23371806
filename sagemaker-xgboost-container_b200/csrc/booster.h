// booster.h -- host-side objects behind the C-ABI handles (DMatrixHandle / BoosterHandle).
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include "container_metrics.h"
#include "curve.h"
#include "engine.h"
#include "grow.h"
#include "json.h"
#include "misc.h"
#include "rank.h"
#include "refresh.h"
#include "sampling.h"
#include "survival.h"
#include "tree.h"

namespace b200 {

// One batch of a QuantileDMatrix as its producer hands it over (upstream's proxy DMatrix): the features stay where the
// producer keeps them until the next batch is requested; the meta information is copied.
struct ProxyBatch {
  enum Kind { kNone, kHostDense, kDevice, kCSR } kind = kNone;
  int64_t n = 0; int F = 0;
  const float* data = nullptr;                        // kHostDense (float32, row-major) / kDevice (float32, C-contiguous)
  std::vector<float> converted;                       // kHostDense of another dtype, converted to float32
  const size_t* indptr = nullptr; const unsigned* indices = nullptr; const float* values = nullptr; size_t nelem = 0;   // kCSR
  std::vector<float> labels, weights, base_margin, label_lower, label_upper;
  int label_cols = 1;                                 // labels is [n][label_cols] row-major
  std::vector<int64_t> qid;
  void clear_meta() { labels.clear(); label_cols = 1; weights.clear(); base_margin.clear(); label_lower.clear(); label_upper.clear(); qid.clear(); }
  void set_float_info(const std::string& field, const float* v, size_t len);
};

// ---------------------------------------------------------------------------------------------
// DMatrix: features resident on the device (raw float row-major + lazily the binned feature blocks)
// ---------------------------------------------------------------------------------------------
class DMatrix {
 public:
  int64_t n = 0; int F = 0;
  bool has_missing = false;
  // a QuantileDMatrix: binned once from batches at construction, X never allocated, the bins fixed at quantile_max_bin
  bool quantile = false; int quantile_max_bin = 0;
  DevBuf<float> X;                                    // n x F, NaN = missing (empty on a quantile matrix)
  std::vector<float> labels, weights, base_margin;    // host copies (returned by GetFloatInfo)
  int label_cols = 1;                                 // T: labels is [n][T] row-major (a multi-target label; 1 from set_float_info)
  DevBuf<float> d_labels, d_weights, d_base_margin;
  std::vector<float> label_lower, label_upper;         // survival:aft interval bounds (label_lower_bound / label_upper_bound)
  DevBuf<float> d_label_lower, d_label_upper;
  CoxOrder cox_order;                                 // survival:cox: the rows sorted by |label|, built on first use, reset with the labels
  // query groups: group g is rows [group_ptr[g], group_ptr[g + 1]) (empty: no groups); under groups a weight is one per group
  std::vector<unsigned> group_ptr;
  RankGroups rank_groups;                             // their device layout, built on first use, reset with the labels, groups or weights
  ContainerSums container_sums;                       // the container metrics' summation plan and label sums (r2), reset with the labels
  std::vector<std::string> feature_names, feature_types;
  // binned representation (built on first use as a training matrix)
  bool binned = false; int binned_max_bin = 0;
  HostCuts cuts; DevBuf<int> d_cut_ptrs; DevBuf<float> d_cut_vals, d_min_vals;
  DevBuf<uint8_t> bins, bins_tail, bins_col, bins_gather; int ngroups = 0, tw = 0, ntail = 0, gather_stride = 0;   // engine.h BinnedMatrix layout
  uint64_t binned_version = 0;                        // bumped by every (re)binning: invalidates captured graphs / cached planes
  uint64_t uid;                                       // identity for prediction caches

  DMatrix();
  static std::unique_ptr<DMatrix> from_dense(const float* data, int64_t nrow, int ncol, float missing);
  static std::unique_ptr<DMatrix> from_device(const float* dptr, int64_t nrow, int ncol, float missing);
  // serving path: CSV text parsed on the device (csv.cu); status 0 ok, 1 ragged rows, 2 needs the host parser
  static std::unique_ptr<DMatrix> from_csv_text(const char* text, int64_t len, char delim, int* status);
  // serving path: libsvm request body parsed on the device (csv.cu); whitespace_mode 0 = tokens split on ' ' (serve_utils),
  // 1 = on any whitespace (encoder); absent = value of entries a line does not list (NaN = missing, or 0); status 0 ok,
  // 2 needs the host route, 3 body without a single entry
  static std::unique_ptr<DMatrix> from_libsvm_text(const char* text, int64_t len, int whitespace_mode, float absent, int* status);
  // training channel: columns label_col / weight_col (-1 = none) become the label / weight info, the rest the features
  static std::unique_ptr<DMatrix> from_csv_text_labeled(const char* text, int64_t len, char delim, int label_col, int weight_col, int* status);
  // columnar input (ingest.cu): `ncols` host column buffers of `nrow` items each, type codes as in include/b200xgb.h; columns
  // label_col / weight_col (-1 = none) become the label / weight info, the others the features in order
  static std::unique_ptr<DMatrix> from_columns(const void* const* cols, const int* types, int ncols, int64_t nrow, int label_col, int weight_col);
  static std::unique_ptr<DMatrix> from_csr(const size_t* indptr, const unsigned* indices, const float* data, size_t nindptr, size_t nelem, size_t ncol);
  // recordio-protobuf body (recordio.cu): status 0 decoded, 1 the body is invalid (*message names the rule), 2 needs the host route
  static std::unique_ptr<DMatrix> from_recordio(const char* buf, int64_t len, int* status, std::string* message);
  // QuantileDMatrix (DESIGN.md "QuantileDMatrix"): reset() then next() until false, twice; next() leaves the batch in *proxy.
  // Cuts: ref's when given, the exact single-rank cuts for one batch, else the multi-rank recipe over the batches in order.
  static std::unique_ptr<DMatrix> from_batches(ProxyBatch* proxy, const std::function<void()>& reset, const std::function<bool()>& next,
                                               DMatrix* ref, float missing, int max_bin);
  // names the reader of the raw features that a quantile matrix cannot serve
  void require_raw(const char* what) const;
  // allow_groups: a matrix with groups may be sliced by whole groups, which the slice carries
  std::unique_ptr<DMatrix> slice(const int* idx, int64_t len, bool allow_groups = false) const;
  void set_float_info(const std::string& field, const float* v, size_t len);
  // a (rows, cols) label, row-major: rows must be the matrix's row count; cols == 1 is the 1-D label
  void set_label_matrix(const float* v, int64_t rows, int64_t cols);
  void set_group_ptr(std::vector<unsigned> ptr);      // validated: starts at 0, non-decreasing, ends at n
  void set_group_sizes(const unsigned* sizes, size_t len);
  void set_qid(const int64_t* qid, size_t len);       // groups are the runs of equal consecutive qid; qid must not decrease
  int64_t num_groups() const { return group_ptr.empty() ? 1 : (int64_t)group_ptr.size() - 1; }
  const std::vector<float>& get_float_info(const std::string& field) const;
  void ensure_binned(int max_bin);
  void set_cuts(const HostCuts& c);                   // external cuts (shared with the oracle in tests)
  BinnedMatrix binned_view() const { BinnedMatrix b; b.bins = bins.p; b.bins_tail = tw ? bins_tail.p : nullptr; b.bins_col = bins_col.p; b.n = n; b.F = F;
    b.bins_gather = bins_gather.p ? bins_gather.p : bins.p; b.gather_stride = gather_stride; b.tail_in_gather = bins_gather.p && tw == 8 ? 1 : 0;
    b.ngroups = ngroups; b.tw = tw; b.ntail = ntail; b.has_missing = has_missing; return b; }
  void finish_upload(float missing);
 private:
  void bin_with_cuts();
  void alloc_bins();                                  // uploads the cuts, allocates the main / tail bins with their pad rows
  void finish_bins();                                 // the aligned and column-major copies of the binned main / tail
};

// device half of DMatrix::from_csr (ingest.cu): X (nrow x F) filled with NaN, then row r's entries [d_ptr[r], d_ptr[r + 1]) stored
// at their indices (an index repeated inside a row keeps its last value); asynchronous on stream s
void csr_to_dense_device(const unsigned long long* d_ptr, const unsigned* d_idx, const float* d_val, int64_t nrow, int F, float* X, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------------------------
struct HostTree {
  std::vector<int> left, right, parent, split_index, split_bin;
  std::vector<uint8_t> default_left;
  std::vector<float> split_cond, base_weight, loss_chg, sum_hess;
  int num_nodes() const { return (int)left.size(); }
};

// process_type=update: the trees to update, taken out of the model at the first update round, and the refresh's device buffers
struct UpdateState {
  bool started = false;
  std::vector<HostTree> trees; std::vector<int> tree_info;
  std::vector<int> indptr{0};                   // layer r = trees [indptr[r], indptr[r + 1])
  std::vector<int> node_off;                    // [trees + 1]: the trees packed one after another
  std::vector<int64_t> block_off;               // [trees]: each tree's result block in out_blocks
  DevBuf<unsigned char> in_block;               // the trees as grow.h tree_block_layout(in_block, total nodes)
  DevBuf<DevNode> nodes; DevBuf<int> d_node_off, d_class; DevBuf<int64_t> d_block_off;
  DevBuf<GH64> sums; DevBuf<int> scratch; DevBuf<unsigned char> out_blocks;
  DevBuf<float2> gpair; DevBuf<unsigned> absmax; DevBuf<float> scales;
  int64_t global_n = 0; uint64_t global_n_uid = 0;   // rows of the job for the matrix with uid global_n_uid
  int layers() const { return (int)indptr.size() - 1; }
};

struct PredCache {
  DevBuf<float> margin; int trees_applied = 0; int64_t n = 0; uint64_t model_version = 0;
  std::vector<float> weights;     // the weight each applied tree was added with (booster=dart changes them after the fact)
};

// booster=dart (upstream DartTrainParam); sample_type 0 uniform / 1 weighted, normalize_type 0 tree / 1 forest
struct DartParam { bool on = false; float rate_drop = 0.0f, skip_drop = 0.0f; int one_drop = 0, sample_type = 0, normalize_type = 0; };

// legacy_io.cc: the pre-JSON binary model format -> the 3.x model document
bool looks_like_legacy_binary(const char* buf, size_t len);
JPtr legacy_binary_to_doc(const char* buf, size_t len);
std::pair<const char*, size_t> legacy_serialized_model_section(const char* buf, size_t len);

class Booster {
 public:
  Booster();
  ~Booster();
  // configuration
  void set_param(const std::string& k, const std::string& v);
  std::string save_config();
  void load_config(const std::string& json);
  // training
  void update_one_iter(int iter, DMatrix* dtrain);
  void boost_one_iter(DMatrix* dtrain, const float* grad, const float* hess, size_t len);
  std::string eval_one_iter(int iter, const std::vector<DMatrix*>& dms, const std::vector<std::string>& names);
  // the raw results of the container's own metrics `names` on dm from the prediction cache (container_metrics.h layout, out
  // holds kContainerOutLen entries); output_margin: the metric reads margins (feval=) instead of predict()'s values
  void eval_container_metrics(DMatrix* dm, const std::vector<std::string>& names, bool output_margin, long long* out);
  // inference; returns host buffer + shape
  void predict(DMatrix* dm, int type, bool training, int iter_begin, int iter_end, bool strict_shape,
               std::vector<float>* out, std::vector<uint64_t>* shape);
  void predict_contribs(DMatrix* dm, int tree_begin, int tree_end, std::vector<float>* out, std::vector<uint64_t>* shape);
  // model IO
  std::string save_model_buffer(const std::string& format);      // "ubj" | "json"
  void load_model_buffer(const char* buf, size_t len);
  std::string serialize();                                         // model + config (pickle)
  void unserialize(const char* buf, size_t len);
  std::unique_ptr<Booster> slice(int begin, int end, int step);
  int boosted_rounds();
  int num_features() const { return num_feature_; }
  std::map<std::string, std::string> attrs;
  std::vector<std::string> feature_names, feature_types;

  // introspection used by tests/bench (build-specific C-ABI entry points)
  void sync_model();                              // materialise pending trees on the host
  void cached_margin(DMatrix* dm, std::vector<float>* out);   // the trainer's prediction cache for dm
  float debug_predict_kernel_ms(DMatrix* dm, int repeats);
  std::string debug_predict_plan(DMatrix* dm, int iter_begin, int iter_end);   // JSON of the plan predict() would run
  const std::vector<HostTree>& trees() { sync_model(); return trees_; }
  const std::vector<int>& tree_info() const { return tree_info_; }
  const std::vector<float>& tree_weights() const { return weight_drop_; }   // all 1 unless booster=dart
  float base_score() const { return base_score_; }
  int num_class() const { return param_.num_class; }
  const TrainParam& param() { configure(); return param_; }
  void set_profile(bool on);
  // the configured objective's gradient pairs at the given host margins [n][K], with round `round`'s row sample; out [n][K][2]
  void debug_gradient(DMatrix* dm, const float* margin, int round, float* out);
  // process_type=update: the (G_q, H_q) sums of every node of the trees being updated (include/b200xgb.h XGB200BoosterGetRefreshSums)
  void debug_refresh_sums(std::vector<long long>* out);
  std::string get_profile();                      // JSON, see include/b200xgb.h
  // histogram of one node for kernel-level parity tests / the roofline bench
  // mode: 0 = production choice (TMA root kernel), 1 = gather kernel, 2 = G-only TMA root kernel (H plane stays zero);
  // + 4 = the training path's tail source, + 8 = G-only payload (g by position, h == 1.0f for every row).
  // row_ids (optional, n_ids entries): histogram of that row subset, gpair given by POSITION -> exercises the gathered path.
  void debug_build_root_hist(DMatrix* dm, const float* gpair_host, std::vector<long long>* hist_out, float* scales_out,
                             int repeats, float* ms_out, int mode = 0, const unsigned* row_ids = nullptr, int64_t n_ids = 0);
  // split evaluation and expansion of a root with the given histogram ([F][256]{g,h} int64) and totals, JSON of every result
  // (include/b200xgb.h XGB200BoosterEvalRootSplit)
  std::string debug_eval_root(DMatrix* dm, const long long* hist_fm, long long G, long long H, float max_g, float max_h,
                              float lower, float upper, const unsigned char* feat_mask);

 private:
  PredictArgs predict_args(DMatrix* dm, int tree_begin, int tree_end);   // the device model on dm (outputs left unset)
  // margins / leaves of trees [pa.tree_begin, pa.tree_end) into pa's outputs: the float predictor, or on a quantile matrix the
  // bin predictor with the model's thresholds mapped to dm's bins first
  void run_predict(DMatrix* dm, PredictArgs pa, cudaStream_t s);
  // predict()'s margins of trees [tb, te) on dm into pred_margin_ (base margin, then the trees; booster=dart: fl(w_t * leaf_t))
  void predict_margin(DMatrix* dm, int tb, int te);
  DevBuf<DevNode> bin_nodes_;                   // d_nodes with each split's cond replaced by its bin threshold (run_predict)
  std::map<std::string, std::string> raw_params_;
  std::vector<std::string> eval_metrics_;
  std::vector<int> monotone_;              // parsed monotone_constraints (empty = none)
  std::vector<std::vector<int>> interaction_;   // parsed interaction_constraints (empty = none)
  bool configured_ = false;
  TrainParam param_;
  std::string objective_name_ = "reg:squarederror";
  bool base_score_set_ = false; float base_score_ = 0.5f; bool base_score_estimated_ = false;
  int num_feature_ = 0;
  int num_target_ = 1;                          // label columns of the model (multi-target regression), fixed by its first round
  std::vector<HostTree> trees_; std::vector<int> tree_info_;
  // boosting round (layer) r holds trees [iteration_indptr_[r], iteration_indptr_[r + 1]): K * num_parallel_tree of them,
  // class-major.  The only round <-> tree map; always starts with 0 and ends with trees_.size()
  std::vector<int> iteration_indptr_{0};
  DevBuf<float2> forest_gpair_;                 // num_parallel_tree > 1 with subsample < 1: the round's unsampled gradients
  GbsScratch gbs_;                              // sampling_method=gradient_based: the threshold select's buffers and thresholds
  std::vector<float> weight_drop_;             // parallel to trees_: the tree's weight in every margin (booster=dart; else 1)
  DartParam dart_;
  float dart_new_weight_ = 1.0f;                // weight of the trees the current dart round grows
  DevBuf<float> dart_drop_margin_;              // the training margin without the round's dropped trees (gradients read it)
  DevBuf<int> dart_ids_; DevBuf<float> dart_coef_;    // tree list and coefficients of the last dart_margin launch
  std::vector<PendingTree> pending_;            // parallel to trees_ (nullptr staging once materialised)
  std::vector<char> on_device_;                 // parallel to trees_: nodes already in d_nodes
  uint64_t model_version_ = 0;
  // device model for prediction
  DevBuf<DevNode> d_nodes; std::vector<int64_t> h_tree_offset; DevBuf<int64_t> d_tree_offset; DevBuf<int> d_tree_info;
  size_t d_nodes_used = 0; int d_trees_uploaded = 0;
  std::map<uint64_t, PredCache> caches_;
  std::unique_ptr<TreeBuilder> builder_ = std::make_unique<TreeBuilder>();   // its device buffers are sized by builder_for
  DevBuf<double> dsum_;                         // device sums of the metrics and of the base-score stump
  CoxScratch cox_scratch_;                      // survival:cox: per-round scratch of the gradient and of cox-nloglik
  RankScratch rank_scratch_;                    // rank:* and the ndcg / map metrics: per-call scratch
  CurveScratch curve_scratch_;                  // aucpr and multi-class auc: per-call scratch, grown on first use
  ContainerScratch container_scratch_;          // the container metrics: per-call scratch, grown on first use
  bool labels_checked_ = false;
  DevBuf<float> pred_margin_, pred_cls_; DevBuf<int> pred_leaf_;      // predict() scratch, grown on demand
  bool children_adjacent_ = true;               // every tree on the device has right child == left child + 1
  // process_type=update: the updaters in order (refresh.h RefreshOp), refresh_leaf, and the trees being updated
  bool update_mode_ = false; std::vector<int> update_ops_; std::string update_ops_str_; int refresh_leaf_ = 1;
  std::unique_ptr<UpdateState> update_ = std::make_unique<UpdateState>();
  DevBuf<float> quantile_alpha_dev_; std::vector<float> quantile_alpha_host_;   // reg:quantileerror / the quantile metric: alpha on the device
  DevBuf<unsigned> target_absmax_;              // reg:quantileerror: each target's max|g| and max h ([2 Q]), for a grid per target

  void configure();
  void check_label_ranges(const DMatrix* dtrain);
  // a matrix's label width against the model: the first round of an empty model takes T from dtrain; the rejections of T > 1
  void check_targets(const DMatrix* dm, bool training);
  const RankGroups& rank_groups(DMatrix* dm, const char* what);   // dm's groups on the device; checks one weight per group
  void begin_update();                               // the model's layers become the trees to update; the model is emptied
  void refresh_one_iter(DMatrix* dtrain);            // one update round: the next layer refreshed / pruned into the model
  int layers() const { return (int)iteration_indptr_.size() - 1; }
  float base_margin() const;
  void estimate_base_score(DMatrix* dtrain);
  void upload_model();
  PredCache& cache_for(DMatrix* dm);
  void bring_cache_up_to_date(DMatrix* dm, PredCache& c);
  void append_device_tree(int class_id, size_t device_offset, int max_nodes, PendingTree pt, float weight);
  std::vector<int> dart_drop_set(int round) const;
  float* dart_begin_round(DMatrix* dtrain, PredCache& c, int round);
  void dart_margin(DMatrix* dm, const std::vector<int>& ids, const std::vector<float>& coef_full, const std::vector<float>& coef_drop,
                   float* m_full, float* m_drop);
  void reserve_nodes(size_t count, size_t slack);    // room for `count` more nodes in d_nodes
  TreeBuilder& builder_for(DMatrix* dm);             // the builder sized for the binned dm and the parameters
  TreeInputs tree_inputs(const DMatrix& dm, const std::string& mask, int tree_index, float* margin, int k);
  void grow_one_tree(DMatrix* dtrain, PredCache& cache, int k, int tree_index);
  // h == 1 for every row in every round on dm: the gradients are a dense float g and the trees grow on it (TreeInputs root_mode)
  bool constant_hessian(const DMatrix& dm) const;
  // sampling_method=gradient_based applies (subsample < 1): the objective writes every row, the trees sample by threshold
  bool gradient_based_sampling() const { return param_.gradient_based && param_.subsample < 1.0f; }
  // tree j of boosting round `round` keeps rows [0, n) of src by the thresholds in gbs_ (launch_gradient_based_sample)
  void gradient_based_sample(const float2* src, float2* dst, int64_t gp_stride, int64_t n, int round, int j, unsigned* absmax);
  void launch_objective(DMatrix* dm, const float* margin, int round, float2* gpair, int64_t gp_stride, unsigned* absmax, float subsample, bool dense_g,
                        float* resid, bool per_target_absmax = false);
  const float* upload_quantile_alpha(const std::vector<float>& alpha);       // the device copy of alpha
  const float* quantile_alpha_device() { return upload_quantile_alpha(param_.quantile_alpha); }
  JPtr model_to_json();
  void model_from_json(const JValue& doc);
  JPtr config_to_json();
  void config_from_json(const JValue& doc);
  void reset_model();
};

// objective name -> engine.h Objective (booster.cu)
const std::map<std::string, int>& objective_table();
// quantile_alpha in any of its accepted forms (booster.cu); raises on a malformed, empty or out-of-range value
std::vector<float> parse_quantile_alpha(const std::string& v);
std::string colsample_mask(unsigned seed, int tree_index, int F, float frac);   // bytes, 1 = feature usable
std::string subset_mask(const std::string& parent, float frac, unsigned seed, uint64_t stream);

}  // namespace b200
