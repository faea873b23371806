// model_io.cc -- Booster model / config (de)serialisation in the xgboost 3.x document schema.
// Serves Booster.save_model / load_model / save_config / pickling as used by the container:
// algorithm_mode/train.py:480-485, serve_utils.py:171-197, serve.py:85-88, checkpointing.py:375,428.
// Schema: SURVEY.md section 8(c) (learner{attributes, feature_names, feature_types, gradient_booster{model{...trees[]}},
// learner_model_param, objective}, version) -- UBJSON for extension-less / .ubj files, JSON text for .json.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include "booster.h"
#include "multi_target.h"

namespace b200 {

static std::string float_repr(float v) {       // shortest round-trip, xgboost style exponent ("1.0026694E1")
  if (std::isnan(v)) return "NaN";
  if (std::isinf(v)) return v > 0 ? "Infinity" : "-Infinity";
  char b[48];
  for (int p = 0; p <= 9; ++p) { snprintf(b, sizeof b, "%.*E", p, (double)v); if (std::strtof(b, nullptr) == v) break; }
  std::string s(b); size_t e = s.find('E');
  std::string mant = s.substr(0, e); int ex = atoi(s.c_str() + e + 1);
  return mant + "E" + std::to_string(ex);
}
static JPtr S(const std::string& s) { return JValue::Str(s); }
// reg:quantileerror's block into raw parameters (read back, and checked, only under that objective by configure)
static void quantile_params_from_json(const JValue& obj, std::map<std::string, std::string>* raw) {
  if (auto qp = obj.get("quantile_loss_param")) if (auto v = qp->get("quantile_alpha")) if (v->type == JValue::kString) (*raw)["quantile_alpha"] = v->s;
}
// the AFT parameter block into raw parameters (read back, and range-checked, only under survival:aft by configure)
static void aft_params_from_json(const JValue& obj, std::map<std::string, std::string>* raw) {
  auto ap = obj.get("aft_loss_param");
  if (!ap) return;
  if (auto v = ap->get("aft_loss_distribution")) (*raw)["aft_loss_distribution"] = v->s;
  if (auto v = ap->get("aft_loss_distribution_scale")) (*raw)["aft_loss_distribution_scale"] = v->type == JValue::kString ? v->s : float_repr((float)v->as_double());
}

// rank:*'s lambdarank_param block into raw parameters (read, and checked, only under those objectives by configure); a field a
// document leaves out keeps its default
static const char* kLambdaRankFields[] = {"lambdarank_pair_method", "lambdarank_num_pair_per_sample", "lambdarank_unbiased", "lambdarank_bias_norm",
                                          "ndcg_exp_gain", "lambdarank_normalization", "lambdarank_score_normalization"};
static void rank_params_from_json(const JValue& obj, std::map<std::string, std::string>* raw) {
  auto lp = obj.get("lambdarank_param");
  if (!lp) return;
  for (const char* f : kLambdaRankFields)
    if (auto v = lp->get(f)) {
      if (v->type == JValue::kString) (*raw)[f] = v->s;
      else if (v->type == JValue::kBool) (*raw)[f] = v->b ? "1" : "0";
      else (*raw)[f] = float_repr((float)v->as_double());
    }
}

// quantile_alpha as "[0.1, 0.5, 0.9]": each value in the fewest %g digits that read back to the same float
static std::string alpha_repr(const std::vector<float>& a) {
  std::string out = "[";
  for (size_t i = 0; i < a.size(); ++i) {
    char b[48];
    for (int p = 1; p <= 9; ++p) { snprintf(b, sizeof b, "%.*g", p, (double)a[i]); if (std::strtof(b, nullptr) == a[i]) break; }
    out += (i ? ", " : "") + std::string(b);
  }
  return out + "]";
}

// per-objective parameter block of the model / config documents (upstream ObjFunction::SaveConfig)
static void objective_params_to_json(JValue& obj, const TrainParam& p) {
  JPtr rp = JValue::Object();
  switch (p.objective) {
    case kPoisson: rp->set("max_delta_step", S(float_repr(p.poisson_max_delta_step))); obj.set("poisson_regression_param", rp); break;
    case kTweedie: rp->set("tweedie_variance_power", S(float_repr(p.tweedie_variance_power))); obj.set("tweedie_regression_param", rp); break;
    case kPseudoHuber: rp->set("huber_slope", S(float_repr(p.huber_slope))); obj.set("pseudo_huber_param", rp); break;
    case kGamma: case kHinge: case kCox: case kAbsoluteError: break;
    case kQuantileError: rp->set("quantile_alpha", S(alpha_repr(p.quantile_alpha))); obj.set("quantile_loss_param", rp); break;   // [UPSTREAM-RECALL]
    case kRankPairwise: case kRankNdcg: case kRankMap: {      // every value a string, as upstream writes them [UPSTREAM-RECALL]
      const std::string v[] = {p.rank_mean ? "mean" : "topk", std::to_string(p.rank_k), p.rank_unbiased ? "1" : "0", float_repr(p.rank_bias_norm), p.rank_exp_gain ? "1" : "0",
                               p.rank_normalization ? "1" : "0", p.rank_score_normalization ? "1" : "0"};
      for (int i = 0; i < 7; ++i) rp->set(kLambdaRankFields[i], S(v[i]));
      obj.set("lambdarank_param", rp); break; }
    case kAft: {
      static const char* dist[] = {"normal", "logistic", "extreme"};
      rp->set("aft_loss_distribution", S(dist[p.aft_dist])); rp->set("aft_loss_distribution_scale", S(float_repr(p.aft_sigma)));
      obj.set("aft_loss_param", rp); break; }
    default: rp->set("scale_pos_weight", S(float_repr(p.scale_pos_weight))); obj.set("reg_loss_param", rp); break;
  }
}

JPtr Booster::model_to_json() {
  configure(); sync_model();
  const int K = param_.num_class;           // classes; the outputs of a quantile model go to num_target
  JPtr doc = JValue::Object();
  JPtr learner = JValue::Object();
  JPtr attributes = JValue::Object();
  for (auto& kv : attrs) attributes->set(kv.first, S(kv.second));
  learner->set("attributes", attributes);
  JPtr fn = JValue::Array(); for (auto& x : feature_names) fn->arr.push_back(S(x)); learner->set("feature_names", fn);
  JPtr ft = JValue::Array(); for (auto& x : feature_types) ft->arr.push_back(S(x)); learner->set("feature_types", ft);
  JPtr gb = JValue::Object(); JPtr model = JValue::Object();
  JPtr gmp = JValue::Object(); gmp->set("num_parallel_tree", S(std::to_string(param_.num_parallel_tree))); gmp->set("num_trees", S(std::to_string(trees_.size())));
  model->set("gbtree_model_param", gmp);
  model->set("iteration_indptr", JValue::I32(std::vector<int32_t>(iteration_indptr_.begin(), iteration_indptr_.end())));
  model->set("tree_info", JValue::I32(std::vector<int32_t>(tree_info_.begin(), tree_info_.end())));
  JPtr trees = JValue::Array();
  for (size_t t = 0; t < trees_.size(); ++t) {
    const HostTree& h = trees_[t]; const int nn = h.num_nodes();
    JPtr tj = JValue::Object();
    tj->set("base_weights", JValue::F32(h.base_weight));
    tj->set("categories", JValue::I32({})); tj->set("categories_nodes", JValue::I32({})); tj->set("categories_segments", JValue::I64({})); tj->set("categories_sizes", JValue::I64({}));
    tj->set("default_left", JValue::U8(h.default_left));
    tj->set("id", JValue::Int((int64_t)t));
    tj->set("left_children", JValue::I32(std::vector<int32_t>(h.left.begin(), h.left.end())));
    tj->set("loss_changes", JValue::F32(h.loss_chg));
    tj->set("parents", JValue::I32(std::vector<int32_t>(h.parent.begin(), h.parent.end())));
    tj->set("right_children", JValue::I32(std::vector<int32_t>(h.right.begin(), h.right.end())));
    tj->set("split_conditions", JValue::F32(h.split_cond));
    tj->set("split_indices", JValue::I32(std::vector<int32_t>(h.split_index.begin(), h.split_index.end())));
    tj->set("split_type", JValue::U8(std::vector<uint8_t>(nn, 0)));
    tj->set("sum_hessian", JValue::F32(h.sum_hess));
    JPtr tp = JValue::Object(); tp->set("num_deleted", S("0")); tp->set("num_feature", S(std::to_string(num_feature_)));
    tp->set("num_nodes", S(std::to_string(nn))); tp->set("size_leaf_vector", S("1"));
    tj->set("tree_param", tp);
    trees->arr.push_back(tj);
  }
  model->set("trees", trees);
  gb->set("model", model); gb->set("name", S("gbtree"));
  if (dart_.on) {            // upstream Dart::SaveModel: the gbtree object under "gbtree", the tree weights beside it
    JPtr dart = JValue::Object(); dart->set("name", S("dart")); dart->set("gbtree", gb);
    dart->set("weight_drop", JValue::F32(std::vector<float>(weight_drop_.begin(), weight_drop_.begin() + trees_.size())));
    gb = dart;
  }
  learner->set("gradient_booster", gb);
  JPtr lmp = JValue::Object();
  // scalar form = the 3.0.x schema this document is stamped with (3.1+ writes the bracketed vector "[1.0E1]", which the
  // reader below accepts as well: the reference's own fixture is a [3,2,0] file)
  lmp->set("base_score", S(float_repr(base_score_))); lmp->set("boost_from_average", S("1"));
  lmp->set("num_class", S(std::to_string(K > 1 ? K : 0))); lmp->set("num_feature", S(std::to_string(num_feature_)));
  lmp->set("num_target", S(std::to_string(param_.objective == kQuantileError ? param_.num_outputs() : param_.num_target)));
  learner->set("learner_model_param", lmp);
  JPtr obj = JValue::Object(); obj->set("name", S(objective_name_));
  if (param_.objective == kSoftprob || param_.objective == kSoftmax) { JPtr sp = JValue::Object(); sp->set("num_class", S(std::to_string(K))); obj->set("softmax_multiclass_param", sp); }
  else objective_params_to_json(*obj, param_);
  learner->set("objective", obj);
  doc->set("learner", learner);
  JPtr ver = JValue::Array(); ver->arr = {JValue::Int(3), JValue::Int(0), JValue::Int(5)};
  doc->set("version", ver);
  return doc;
}

void Booster::reset_model() {
  sync_model();
  trees_.clear(); tree_info_.clear(); iteration_indptr_.assign(1, 0); weight_drop_.clear(); pending_.clear(); on_device_.clear(); h_tree_offset.clear();
  d_nodes_used = 0; d_trees_uploaded = 0; caches_.clear(); ++model_version_; children_adjacent_ = true;
}

template <typename T, typename F> static std::vector<T> num_vec(const JValue& a, F conv) {
  std::vector<T> v(a.length()); for (size_t i = 0; i < v.size(); ++i) v[i] = conv(a.num_at(i)); return v;
}

void Booster::model_from_json(const JValue& doc) {
  const JValue& learner = doc.at("learner");
  reset_model();
  update_ = std::make_unique<UpdateState>();     // process_type=update starts over from the loaded trees
  attrs.clear();
  if (auto a = learner.get("attributes")) for (auto& kv : a->obj) attrs[kv.first] = kv.second->s;
  feature_names.clear(); feature_types.clear();
  if (auto a = learner.get("feature_names")) for (auto& x : a->arr) feature_names.push_back(x->s);
  if (auto a = learner.get("feature_types")) for (auto& x : a->arr) feature_types.push_back(x->s);
  const JValue& obj = learner.at("objective");
  objective_name_ = obj.at("name").s;
  raw_params_["objective"] = objective_name_;
  if (auto rp = obj.get("reg_loss_param")) if (auto sp = rp->get("scale_pos_weight")) raw_params_["scale_pos_weight"] = std::to_string(sp->as_double());
  if (auto pp = obj.get("poisson_regression_param")) if (auto v = pp->get("max_delta_step")) raw_params_["max_delta_step"] = std::to_string(v->as_double());
  if (auto tp = obj.get("tweedie_regression_param")) if (auto v = tp->get("tweedie_variance_power")) raw_params_["tweedie_variance_power"] = std::to_string(v->as_double());
  if (auto hp = obj.get("pseudo_huber_param")) if (auto v = hp->get("huber_slope")) raw_params_["huber_slope"] = std::to_string(v->as_double());
  aft_params_from_json(obj, &raw_params_);
  quantile_params_from_json(obj, &raw_params_);
  rank_params_from_json(obj, &raw_params_);
  const JValue& lmp = learner.at("learner_model_param");
  num_feature_ = (int)lmp.at("num_feature").as_int();
  int nc = lmp.has("num_class") ? (int)lmp.at("num_class").as_int() : 0;
  if (nc > 1) raw_params_["num_class"] = std::to_string(nc);
  else if (auto sp = obj.get("softmax_multiclass_param")) raw_params_["num_class"] = std::to_string((int)sp->at("num_class").as_int());
  base_score_ = (float)lmp.at("base_score").as_double(); base_score_set_ = true; base_score_estimated_ = true;
  raw_params_.erase("base_score");
  configured_ = false;
  const JValue* gbp = &learner.at("gradient_booster");
  const std::string gb_name = gbp->at("name").s;
  B200_CHECK(gb_name == "gbtree" || gb_name == "dart", "Only gbtree and dart models can be loaded (got " + gb_name + ")");
  const JValue* weights = nullptr;
  if (gb_name == "dart") { weights = &gbp->at("weight_drop"); gbp = &gbp->at("gbtree"); raw_params_["booster"] = "dart"; }
  else if (raw_params_.count("booster") && raw_params_["booster"] == "dart") raw_params_.erase("booster");
  const JValue& gb = *gbp;
  const JValue& model = gb.at("model");
  const JValue& trees = model.at("trees");
  const JValue& tinfo = model.at("tree_info");
  B200_CHECK(trees.type == JValue::kArray && tinfo.length() == trees.arr.size(), "model: tree_info does not have one entry per tree");
  int K = std::max(1, nc); if (nc <= 1) if (auto sp = obj.get("softmax_multiclass_param")) K = std::max(1, (int)sp->at("num_class").as_int());
  if (objective_name_ == "reg:quantileerror") {   // one output per quantile_alpha entry: num_target of them
    const int nt = lmp.has("num_target") ? (int)lmp.at("num_target").as_int() : 1;
    auto qa = raw_params_.find("quantile_alpha");
    B200_CHECK(qa != raw_params_.end(), "model: a reg:quantileerror model needs objective.quantile_loss_param.quantile_alpha");
    B200_CHECK((int)parse_quantile_alpha(qa->second).size() == nt, "model: num_target is " + std::to_string(nt) + " but quantile_alpha is " + qa->second);
    K = std::max(1, nt);
  }
  // multi-target regression: num_target outputs of one of the multi-target objectives (multi_target.h)
  num_target_ = 1;
  if (objective_name_ != "reg:quantileerror" && lmp.has("num_target")) {
    const int64_t nt = lmp.at("num_target").as_int();
    B200_CHECK(nt >= 1 && nt <= (1 << 20), "model: num_target must be a positive integer (got " + std::to_string(nt) + ")");
    auto ot = objective_table().find(objective_name_);
    B200_CHECK(nt == 1 || (ot != objective_table().end() && objective_is_multi_target(ot->second)), "model: num_target is " + std::to_string(nt) +
               " but objective " + objective_name_ + " does not support multi-target models (multi-target)");
    B200_CHECK(nt == 1 || nc <= 1, "model: num_target and num_class cannot both be above 1");
    num_target_ = (int)nt;
    if (nt > 1) K = (int)nt;
  }
  for (size_t t = 0; t < trees.arr.size(); ++t) { const double g = tinfo.num_at(t); B200_CHECK(g >= 0 && g < K, "model: tree_info entry out of range"); }
  // the layer layout: iteration_indptr when the document has it (2.x / 3.x), else K * num_parallel_tree trees per round (1.x)
  int P = 1;
  if (auto gmp = model.get("gbtree_model_param")) if (auto v = gmp->get("num_parallel_tree")) {
    const double d = v->as_double();
    B200_CHECK(d >= 1.0 && d <= (double)(1 << 20) && d == std::floor(d), "model: num_parallel_tree must be a positive integer");
    P = (int)d;
  }
  const int64_t ntrees = (int64_t)trees.arr.size();
  std::vector<int> indptr;
  if (auto ip = model.get("iteration_indptr")) {
    B200_CHECK(ip->length() >= 1, "model: iteration_indptr is empty");
    for (size_t r = 0; r < ip->length(); ++r) {
      const double v = ip->num_at(r);
      B200_CHECK(v == std::floor(v) && v >= 0 && v <= (double)ntrees, "model: iteration_indptr entry " + std::to_string(r) + " is not a tree count in [0, " + std::to_string(ntrees) + "]");
      B200_CHECK(r > 0 || v == 0, "model: iteration_indptr must start with 0");
      B200_CHECK(r == 0 || (int)v >= indptr.back(), "model: iteration_indptr must not decrease");
      indptr.push_back((int)v);
    }
    B200_CHECK(indptr.back() == ntrees, "model: iteration_indptr ends at " + std::to_string(indptr.back()) + " but the model has " + std::to_string(ntrees) + " trees");
  } else {
    const int64_t per = (int64_t)K * P;
    B200_CHECK(ntrees % per == 0, "model: " + std::to_string(ntrees) + " trees are not whole rounds of num_class x num_parallel_tree = " + std::to_string(per));
    for (int64_t t = 0; t <= ntrees; t += per) indptr.push_back((int)t);
  }
  iteration_indptr_ = indptr;
  raw_params_["num_parallel_tree"] = std::to_string(P);
  for (size_t t = 0; t < trees.arr.size(); ++t) {
    const JValue& tj = *trees.arr[t];
    HostTree h;
    auto toi = [](double x) { return (int)x; }; auto tof = [](double x) { return (float)x; }; auto tou = [](double x) { return (uint8_t)x; };
    h.left = num_vec<int>(tj.at("left_children"), toi); h.right = num_vec<int>(tj.at("right_children"), toi);
    h.parent = num_vec<int>(tj.at("parents"), toi); h.split_index = num_vec<int>(tj.at("split_indices"), toi);
    h.default_left = num_vec<uint8_t>(tj.at("default_left"), tou);
    h.split_cond = num_vec<float>(tj.at("split_conditions"), tof); h.base_weight = num_vec<float>(tj.at("base_weights"), tof);
    h.loss_chg = num_vec<float>(tj.at("loss_changes"), tof); h.sum_hess = num_vec<float>(tj.at("sum_hessian"), tof);
    h.split_bin.assign(h.left.size(), -1);
    if (auto st = tj.get("split_type")) for (size_t i = 0; i < st->length(); ++i) B200_CHECK(st->num_at(i) == 0, "categorical splits are not supported on the B200 path");
    const size_t nn = h.left.size();
    B200_CHECK(h.right.size() == nn && h.split_index.size() == nn && h.split_cond.size() == nn && h.default_left.size() == nn, "model: inconsistent tree array lengths");
    B200_CHECK(nn >= 1 && h.parent.size() == nn && h.base_weight.size() == nn && h.loss_chg.size() == nn && h.sum_hess.size() == nn, "model: inconsistent tree array lengths");
    // the device kernels walk these arrays unchecked: children must exist and lie AFTER their parent (xgboost allocates node ids
    // in expansion order), which also rules out cycles; split features must exist
    for (size_t i = 0; i < nn; ++i) {
      const int l = h.left[i], r = h.right[i];
      if (l == -1 && r == -1) continue;
      B200_CHECK(l > (int)i && r > (int)i && (size_t)l < nn && (size_t)r < nn && l != r, "model: tree " + std::to_string(t) + " node " + std::to_string(i) + " has child indices out of order or out of range");
      B200_CHECK(h.split_index[i] >= 0 && h.split_index[i] < std::max(num_feature_, 1), "model: tree " + std::to_string(t) + " node " + std::to_string(i) + " splits on feature " + std::to_string(h.split_index[i]) + " but the model has " + std::to_string(num_feature_) + " features");
    }
    trees_.push_back(std::move(h)); tree_info_.push_back((int)tinfo.num_at(t)); pending_.emplace_back(); on_device_.push_back(0);
  }
  weight_drop_.assign(trees_.size(), 1.0f);
  if (weights) {             // a typed f32 array or a plain numeric array, one finite weight per tree
    B200_CHECK(weights->type == JValue::kF32Array || weights->type == JValue::kArray, "model: weight_drop must be an array of numbers");
    B200_CHECK(weights->length() == trees_.size(), "model: weight_drop has " + std::to_string(weights->length()) + " entries for " + std::to_string(trees_.size()) + " trees");
    for (size_t t = 0; t < trees_.size(); ++t) {
      const double w = weights->num_at(t);
      B200_CHECK(std::isfinite(w) && std::isfinite((float)w), "model: weight_drop entry " + std::to_string(t) + " is not finite");
      weight_drop_[t] = (float)w;
    }
  }
  ++model_version_;
}

std::string Booster::save_model_buffer(const std::string& format) {
  JPtr doc = model_to_json();
  std::string out;
  if (format == "json") json_write(*doc, &out); else ubj_write(*doc, &out);
  return out;
}

static JPtr parse_any(const char* buf, size_t len) {
  B200_CHECK(len >= 2, "model buffer is empty");
  size_t i = 0; while (i < len && (buf[i] == ' ' || buf[i] == '\n' || buf[i] == '\t' || buf[i] == '\r')) ++i;
  B200_CHECK(i < len && buf[i] == '{', "Unknown model format: expected an xgboost JSON / UBJSON document or a legacy binary model");
  char c = i + 1 < len ? buf[i + 1] : 0;
  if (c == '"' || c == ' ' || c == '\n' || c == '\t' || c == '\r' || c == '}') return JsonReader(buf + i, len - i).parse();
  return UbjReader(reinterpret_cast<const unsigned char*>(buf + i), len - i).parse();
}

void Booster::load_model_buffer(const char* buf, size_t len) {
  // pre-JSON binary files and the pickled state of xgboost 1.x Boosters (serve_utils.py:171-197 meets both): legacy_io.cc
  auto sect = legacy_serialized_model_section(buf, len);
  if (sect.first != nullptr) { model_from_json(*legacy_binary_to_doc(sect.first, sect.second)); return; }   // (its 1.x config section names only defaults)
  if (looks_like_legacy_binary(buf, len)) { model_from_json(*legacy_binary_to_doc(buf, len)); return; }
  JPtr doc = parse_any(buf, len);
  if (doc->has("Model")) { model_from_json(doc->at("Model")); if (doc->has("Config")) config_from_json(doc->at("Config")); }
  else model_from_json(*doc);
}

// ---- config (Booster.save_config): the container reads learner.objective.name and learner.learner_model_param.num_class
JPtr Booster::config_to_json() {
  configure();
  JPtr doc = JValue::Object(); JPtr learner = JValue::Object();
  JPtr gp = JValue::Object(); gp->set("device", S("cuda:0")); gp->set("seed", S(std::to_string(param_.seed))); gp->set("nthread", S("0"));
  learner->set("generic_param", gp);
  JPtr gb = JValue::Object(); gb->set("name", S("gbtree"));
  JPtr gmp = JValue::Object(); gmp->set("num_parallel_tree", S(std::to_string(param_.num_parallel_tree))); gmp->set("num_trees", S(std::to_string(trees_.size()))); gb->set("gbtree_model_param", gmp);
  JPtr gtp = JValue::Object(); gtp->set("process_type", S(update_mode_ ? "update" : "default")); gtp->set("tree_method", S("hist"));
  gtp->set("updater", S(update_mode_ ? update_ops_str_ : "grow_b200_hist")); gb->set("gbtree_train_param", gtp);
  JPtr ttp = JValue::Object();
  auto f = [&](const char* k, float v) { ttp->set(k, S(float_repr(v))); }; auto i = [&](const char* k, int v) { ttp->set(k, S(std::to_string(v))); };
  f("alpha", param_.alpha); f("colsample_bylevel", param_.colsample_bylevel); f("colsample_bynode", param_.colsample_bynode); f("colsample_bytree", param_.colsample_bytree);
  f("eta", param_.eta); f("gamma", param_.gamma); ttp->set("grow_policy", S(param_.lossguide ? "lossguide" : "depthwise")); f("lambda", param_.lambda); i("max_bin", param_.max_bin);
  f("max_delta_step", param_.max_delta_step); i("max_depth", param_.max_depth); i("max_leaves", param_.max_leaves); f("min_child_weight", param_.min_child_weight);
  f("subsample", param_.subsample); ttp->set("sampling_method", S(param_.gradient_based ? "gradient_based" : "uniform"));
  if (update_mode_) i("refresh_leaf", refresh_leaf_);
  if (!monotone_.empty()) { std::string v = "("; for (size_t j = 0; j < monotone_.size(); ++j) { if (j) v += ","; v += std::to_string(monotone_[j]); } v += ")"; ttp->set("monotone_constraints", S(v)); }
  if (!interaction_.empty()) {
    std::string v = "[";
    for (size_t si = 0; si < interaction_.size(); ++si) { v += si ? ",[" : "["; for (size_t j = 0; j < interaction_[si].size(); ++j) { if (j) v += ","; v += std::to_string(interaction_[si][j]); } v += "]"; }
    v += "]"; ttp->set("interaction_constraints", S(v));
  }
  gb->set("tree_train_param", ttp);
  if (dart_.on) {            // upstream Dart::SaveConfig: {"name": "dart", "dart_train_param": {...}, "gbtree": {<gbtree config>}}
    JPtr dart = JValue::Object(); dart->set("name", S("dart"));
    JPtr dtp = JValue::Object();
    dtp->set("normalize_type", S(dart_.normalize_type == 1 ? "forest" : "tree")); dtp->set("one_drop", S(dart_.one_drop ? "1" : "0"));
    dtp->set("rate_drop", S(float_repr(dart_.rate_drop))); dtp->set("sample_type", S(dart_.sample_type == 1 ? "weighted" : "uniform"));
    dtp->set("skip_drop", S(float_repr(dart_.skip_drop)));
    dart->set("dart_train_param", dtp); dart->set("gbtree", gb);
    gb = dart;
  }
  learner->set("gradient_booster", gb);
  JPtr lmp = JValue::Object(); lmp->set("base_score", S(float_repr(base_score_))); lmp->set("boost_from_average", S("1"));
  lmp->set("num_class", S(std::to_string(param_.num_class > 1 ? param_.num_class : 0))); lmp->set("num_feature", S(std::to_string(num_feature_)));
  lmp->set("num_target", S(std::to_string(param_.objective == kQuantileError ? param_.num_outputs() : param_.num_target)));
  learner->set("learner_model_param", lmp);
  JPtr ltp = JValue::Object(); ltp->set("booster", S(dart_.on ? "dart" : "gbtree")); ltp->set("disable_default_eval_metric", S("0")); ltp->set("multi_strategy", S("one_output_per_tree")); ltp->set("objective", S(objective_name_));
  learner->set("learner_train_param", ltp);
  JPtr metrics = JValue::Array(); for (auto& m : eval_metrics_) { JPtr mo = JValue::Object(); mo->set("name", S(m)); metrics->arr.push_back(mo); } learner->set("metrics", metrics);
  JPtr obj = JValue::Object(); obj->set("name", S(objective_name_));
  if (param_.objective == kSoftprob || param_.objective == kSoftmax) { JPtr sp = JValue::Object(); sp->set("num_class", S(std::to_string(param_.num_class))); obj->set("softmax_multiclass_param", sp); }
  else objective_params_to_json(*obj, param_);
  learner->set("objective", obj);
  doc->set("learner", learner);
  JPtr ver = JValue::Array(); ver->arr = {JValue::Int(3), JValue::Int(0), JValue::Int(5)}; doc->set("version", ver);
  return doc;
}

void Booster::config_from_json(const JValue& doc) {
  const JValue& learner = doc.at("learner");
  if (auto gb = learner.get("gradient_booster")) {
    if (gb->get("name") && gb->at("name").s == "dart") {
      raw_params_["booster"] = "dart";
      if (auto dtp = gb->get("dart_train_param")) for (auto& kv : dtp->obj) if (kv.second->type == JValue::kString) raw_params_[kv.first] = kv.second->s;
      if (auto inner = gb->get("gbtree")) gb = inner;
    }
    if (auto ttp = gb->get("tree_train_param")) for (auto& kv : ttp->obj) if (kv.second->type == JValue::kString) raw_params_[kv.first] = kv.second->s;
    if (auto gtp = gb->get("gbtree_train_param")) if (auto pt = gtp->get("process_type")) if (pt->type == JValue::kString && pt->s == "update") {
      raw_params_["process_type"] = "update";          // the default mode's gbtree_train_param names this engine's own updater
      if (auto up = gtp->get("updater")) if (up->type == JValue::kString) raw_params_["updater"] = up->s;
    }
    if (auto gmp = gb->get("gbtree_model_param")) if (auto v = gmp->get("num_parallel_tree")) if (v->type == JValue::kString) raw_params_["num_parallel_tree"] = v->s;
  }
  if (auto gp = learner.get("generic_param")) if (auto sd = gp->get("seed")) raw_params_["seed"] = sd->s;
  if (auto o = learner.get("objective")) {
    raw_params_["objective"] = o->at("name").s;
    if (auto rp = o->get("reg_loss_param")) if (auto sp = rp->get("scale_pos_weight")) raw_params_["scale_pos_weight"] = sp->s;
    if (auto sp = o->get("softmax_multiclass_param")) raw_params_["num_class"] = sp->at("num_class").s;
    if (auto pp = o->get("poisson_regression_param")) if (auto v = pp->get("max_delta_step")) raw_params_["max_delta_step"] = v->s;
    if (auto tp = o->get("tweedie_regression_param")) if (auto v = tp->get("tweedie_variance_power")) raw_params_["tweedie_variance_power"] = v->s;
    if (auto hp = o->get("pseudo_huber_param")) if (auto v = hp->get("huber_slope")) raw_params_["huber_slope"] = v->s;
    aft_params_from_json(*o, &raw_params_);
    quantile_params_from_json(*o, &raw_params_);
    rank_params_from_json(*o, &raw_params_);
    // a multi-target model's num_target (the model document carries it too; a fresh Booster takes it from the config)
    if (auto lmp = learner.get("learner_model_param")) if (auto nt = lmp->get("num_target")) if (nt->type == JValue::kString && o->at("name").s != "reg:quantileerror") {
      auto ot = objective_table().find(o->at("name").s);
      const int v = std::atoi(nt->s.c_str());
      if (v > 1) B200_CHECK(ot != objective_table().end() && objective_is_multi_target(ot->second), "config: num_target is " + nt->s + " but objective " +
                            o->at("name").s + " does not support multi-target models (multi-target)");
      if (v >= 1) num_target_ = v;
    }
  }
  if (auto m = learner.get("metrics")) { eval_metrics_.clear(); for (auto& x : m->arr) eval_metrics_.push_back(x->at("name").s); }
  configured_ = false;
}

std::string Booster::save_config() { std::string out; json_write(*config_to_json(), &out); return out; }
void Booster::load_config(const std::string& json) { config_from_json(*parse_json(json)); }

std::string Booster::serialize() {
  JPtr doc = JValue::Object(); doc->set("Model", model_to_json()); doc->set("Config", config_to_json());
  std::string out; ubj_write(*doc, &out); return out;
}
void Booster::unserialize(const char* buf, size_t len) { load_model_buffer(buf, len); }

std::unique_ptr<Booster> Booster::slice(int begin, int end, int step) {
  configure(); sync_model();
  const int rounds = layers();
  if (end == 0) end = rounds;
  B200_CHECK(step >= 1, "Invalid slice step");
  B200_CHECK(begin >= 0 && begin < end && end <= rounds, "Layer index out of range");     // upstream message for an empty / OOB slice
  auto b = std::make_unique<Booster>();
  b->raw_params_ = raw_params_; b->eval_metrics_ = eval_metrics_; b->attrs = attrs; b->feature_names = feature_names; b->feature_types = feature_types;
  b->objective_name_ = objective_name_; b->base_score_ = base_score_; b->base_score_set_ = base_score_set_; b->base_score_estimated_ = true; b->num_feature_ = num_feature_;
  b->num_target_ = num_target_;
  b->raw_params_.erase("base_score"); b->base_score_set_ = true;
  for (int r = begin; r < end; r += step) {
    for (int t = iteration_indptr_[r]; t < iteration_indptr_[r + 1]; ++t) {
      b->trees_.push_back(trees_[t]); b->tree_info_.push_back(tree_info_[t]); b->weight_drop_.push_back(weight_drop_[t]);
      b->pending_.emplace_back(); b->on_device_.push_back(0);
    }
    b->iteration_indptr_.push_back((int)b->trees_.size());
  }
  return b;
}

}  // namespace b200
