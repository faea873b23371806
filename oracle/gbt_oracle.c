/*
 * gbt_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the `tree_method=hist` boosting path that the reference container
 * (aws/sagemaker-xgboost-container) reaches through `xgb.train` / `Booster.predict`
 *   - call sites: src/sagemaker_xgboost_container/algorithm_mode/train.py:367-376,432-442
 *                 src/sagemaker_xgboost_container/algorithm_mode/serve_utils.py:244-250
 * The arithmetic itself lives in the third-party wheel xgboost==3.0.5
 * (docker/3.0-5/base/Dockerfile.cpu:33,212), which is NOT vendored in /root/reference and not
 * installable here.  This file restates the published algorithm of dmlc/xgboost v3.0.5 from recall
 * ("[UPSTREAM-RECALL]" in SURVEY.md section 8); each function names the upstream file it follows.
 *
 * PARITY STATUS: pinned on two models the real library trained, both held by the reference's own tests:
 *   (1) WHOLE MODEL -- test/resources/models/saved_booster/xgboost-model is xgboost's 20-round multi:softprob run on the
 *       150-row iris data (eta 0.3, max_depth 3, lambda 1): this file re-trains it and reproduces all 60 trees -- structure,
 *       split features, the partition of the rows at every node, loss_chg / cover / leaf values to float32 round-off
 *       (tests/test_iris_real_xgboost_pin.py; the CUDA path passes the same test).  What that run does not exercise stays
 *       pinned at formula level only: missing values, sample weights, quantile cuts beyond 256 distinct values, row / column
 *       sampling (own RNG), the objectives other than softmax.
 *   (2) FORMULAS -- test/resources/abalone/models/libsvm_pickled/xgboost-model (tests/test_oracle_fixture.py): gain and weight
 *       on its 715 nodes, leaf = eta*w, gamma / min_child_weight thresholds, base score, traversal rule x < thr -> left.
 *   No xgboost binary exists in this image; nothing else can be run against the real library.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
 * load this library.
 *
 * Build: gcc -O3 -fopenmp -fPIC -shared -o oracle/libgbt_oracle.so oracle/gbt_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_MISSING_BIN 255
#define K_RT_EPS 1e-6f

enum { OBJ_SQUAREDERROR = 0, OBJ_BINARY_LOGISTIC = 1, OBJ_REG_LOGISTIC = 2, OBJ_LOGITRAW = 3,
       OBJ_SOFTPROB = 4, OBJ_SOFTMAX = 5,
       OBJ_SQUAREDLOGERROR = 6, OBJ_PSEUDOHUBER = 7, OBJ_POISSON = 8, OBJ_GAMMA = 9, OBJ_TWEEDIE = 10, OBJ_HINGE = 11 };

typedef struct {
  int32_t objective;
  int32_t num_class;        /* 1 unless multi:* */
  int32_t max_depth;        /* 0 = unlimited */
  int32_t max_leaves;       /* 0 = unlimited */
  int32_t max_bin;
  int32_t grow_policy;      /* 0 depthwise, 1 lossguide */
  int32_t nthread;
  uint32_t seed;
  float eta, lambda, alpha, gamma, min_child_weight, max_delta_step, scale_pos_weight;
  float subsample, colsample_bytree, colsample_bylevel, colsample_bynode;
  float huber_slope, tweedie_variance_power, poisson_max_delta_step;    /* objective parameters (upstream defaults 1, 1.5, 0.7) */
} OrcParams;

/* ------------------------------------------------------------------------------------------ */
/* Quantile cuts.  [UPSTREAM src/common/hist_util.cc, quantile.cc]                              */
/* Upstream runs a weighted GK sketch; that cannot be restated bit-exactly without source, so   */
/* both the oracle and the product define cuts from EXACT weighted quantiles over the sorted    */
/* distinct values.  Identical to upstream whenever a feature has <= max_bin distinct values:   */
/*   cuts = {distinct[1..m-1]} U {last + (|last| + 1e-5)},  min_val = min - (|min| + 1e-5)      */
/*   bin(v) = upper_bound(cuts, v) clipped to the last bin; NaN -> ORC_MISSING_BIN.             */
/* ------------------------------------------------------------------------------------------ */
typedef struct { float v; float w; } VW;
static int cmp_vw(const void* a, const void* b) {
  float x = ((const VW*)a)->v, y = ((const VW*)b)->v;
  return (x > y) - (x < y);
}

/* Shared definition (mirrored by csrc/quantile.cu): given the m distinct sorted values d[] with
 * total weights cw[] of one feature, emit at most `nb` cuts.  Returns the number of cuts. */
static int cuts_from_distinct(const float* d, const double* cw, int64_t m, int nb, float* out) {
  int nc = 0;
  if (m == 0) { out[0] = 1e-5f; return 1; }     /* feature entirely missing: one dummy bin */
  if (m <= nb) {
    for (int64_t i = 1; i < m; ++i) out[nc++] = d[i];
  } else {
    /* exact weighted quantiles: for k = 1..nb-1 pick the first distinct value whose cumulative
     * weight (inclusive) reaches k*W/nb; the cut is the NEXT distinct value's lower edge, i.e.
     * the value itself (bin = upper_bound), deduplicated and strictly increasing. */
    double W = 0; for (int64_t i = 0; i < m; ++i) W += cw[i];
    double cum = 0; int64_t i = 0; float last = d[0];
    for (int k = 1; k < nb; ++k) {
      double target = W * (double)k / (double)nb;
      while (i < m && cum + cw[i] < target) { cum += cw[i]; ++i; }
      /* d[i] is the value at which the running weight crosses target; cut after it */
      int64_t j = i + 1 < m ? i + 1 : m - 1;
      float c = d[j];
      if (c > last) { out[nc++] = c; last = c; }
    }
  }
  float lastv = d[m - 1];
  out[nc++] = lastv + (fabsf(lastv) + 1e-5f);
  return nc;
}

/* X row-major n x F (NaN = missing). w may be NULL. max_bin_eff = max_bin, or 255 if the matrix
 * has missing values (bin code 255 is reserved for "missing" in the uint8 layout).
 * cut_ptrs: F+1 ints; cut_vals: capacity F*max_bin; min_vals: F. Returns total number of cuts. */
int orc_make_cuts(const float* X, int64_t n, int32_t F, const float* w, int32_t max_bin,
                  int32_t* cut_ptrs, float* cut_vals, float* min_vals, int32_t* has_missing_out) {
  int has_missing = 0;
  for (int64_t i = 0; i < n * (int64_t)F && !has_missing; ++i) if (isnan(X[i])) has_missing = 1;
  if (has_missing_out) *has_missing_out = has_missing;
  int nb = max_bin;
  if (nb > 256) nb = 256;
  if (has_missing && nb > 255) nb = 255;
  /* features are independent: sort / collapse them in parallel into per-feature cut lists, then concatenate */
  float* tmp_cuts = (float*)malloc(sizeof(float) * (size_t)F * 256);
  int* tmp_n = (int*)malloc(sizeof(int) * (size_t)(F > 0 ? F : 1));
#pragma omp parallel
  {
    VW* col = (VW*)malloc(sizeof(VW) * (size_t)(n > 0 ? n : 1));
    float* d = (float*)malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
    double* cw = (double*)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
#pragma omp for schedule(dynamic, 1)
    for (int f = 0; f < F; ++f) {
      int64_t cnt = 0;
      for (int64_t r = 0; r < n; ++r) {
        float v = X[r * F + f];
        if (!isnan(v)) { col[cnt].v = v; col[cnt].w = w ? w[r] : 1.0f; ++cnt; }
      }
      qsort(col, (size_t)cnt, sizeof(VW), cmp_vw);
      int64_t m = 0;
      for (int64_t i = 0; i < cnt; ++i) {
        if (m > 0 && col[i].v == d[m - 1]) cw[m - 1] += col[i].w;
        else { d[m] = col[i].v; cw[m] = col[i].w; ++m; }
      }
      tmp_n[f] = cuts_from_distinct(d, cw, m, nb, tmp_cuts + (size_t)f * 256);
      float mn = m > 0 ? d[0] : 0.0f;
      min_vals[f] = mn - (fabsf(mn) + 1e-5f);
    }
    free(col); free(d); free(cw);
  }
  int total = 0;
  cut_ptrs[0] = 0;
  for (int f = 0; f < F; ++f) {
    memcpy(cut_vals + total, tmp_cuts + (size_t)f * 256, sizeof(float) * (size_t)tmp_n[f]);
    total += tmp_n[f];
    cut_ptrs[f + 1] = total;
  }
  free(tmp_cuts); free(tmp_n);
  return total;
}

/* [UPSTREAM src/data/gradient_index.cc, src/common/hist_util.h SearchBin] */
void orc_bin(const float* X, int64_t n, int32_t F, const int32_t* cut_ptrs, const float* cut_vals,
             uint8_t* bins) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n; ++r) {
    for (int f = 0; f < F; ++f) {
      float v = X[r * F + f];
      uint8_t b;
      if (isnan(v)) b = ORC_MISSING_BIN;
      else {
        const float* c = cut_vals + cut_ptrs[f];
        int nc = cut_ptrs[f + 1] - cut_ptrs[f];
        int lo = 0, hi = nc;              /* upper_bound: first cut > v */
        while (lo < hi) { int mid = (lo + hi) >> 1; if (c[mid] > v) hi = mid; else lo = mid + 1; }
        if (lo >= nc) lo = nc - 1;
        b = (uint8_t)lo;
      }
      bins[r * F + f] = b;
    }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* Objective.  [UPSTREAM src/objective/regression_loss.h, regression_obj.cu, multiclass_obj.cu] */
/* ------------------------------------------------------------------------------------------ */
static inline float orc_sigmoid(float x) {
  const float kEps = 1e-16f;
  x = fminf(-x, 88.7f);
  float denom = expf(x) + 1.0f + kEps;
  return 1.0f / denom;
}

/* margins: n x K row-major; gpair out: n x K x 2 (g,h) row-major.  Returns 0, or a negative code
 * for a label error (-1 logistic label range, -2 multiclass label range, -3 squaredlogerror label <= -1, -4 poisson label < 0,
 * -5 gamma label <= 0, -6 tweedie label < 0).
 * Formulas [UPSTREAM-RECALL v3.0.5]: regression_loss.h (LinearSquareLoss, LogisticRegression, SquaredLogError, PseudoHuberError via
 * regression_obj.cu), regression_obj.cu (PoissonRegression: hess = exp(p + max_delta_step); GammaRegression; TweedieRegression),
 * hinge.cu (y' = 2y - 1; p*y' < 1 ? (-y', 1) : (0, FLT_MIN)).  scale_pos_weight belongs to the RegLossObj family only. */
int orc_gradient(const OrcParams* p, const float* margins, const float* labels, const float* weights,
                 int64_t n, float* gpair) {
  const int K = p->num_class > 1 ? p->num_class : 1;
  int err = 0;
  if (p->objective == OBJ_SOFTPROB || p->objective == OBJ_SOFTMAX) {
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < n; ++r) {
      const float* m = margins + r * K;
      float wmax = m[0];
      for (int k = 1; k < K; ++k) wmax = fmaxf(wmax, m[k]);
      float wsum = 0.0f;
      for (int k = 0; k < K; ++k) wsum += expf(m[k] - wmax);
      float w = weights ? weights[r] : 1.0f;
      int label = (int)labels[r];
      if (label < 0 || label >= K) { err = -2; label = 0; }
      for (int k = 0; k < K; ++k) {
        float pk = expf(m[k] - wmax) / wsum;
        const float eps = 1e-16f;
        float h = fmaxf(2.0f * pk * (1.0f - pk) * w, eps);
        float g = (label == k ? pk - 1.0f : pk) * w;
        gpair[(r * K + k) * 2 + 0] = g;
        gpair[(r * K + k) * 2 + 1] = h;
      }
    }
    return err;
  }
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n; ++r) {
    float y = labels[r];
    float w = weights ? weights[r] : 1.0f;
    const int reg_loss = p->objective <= OBJ_LOGITRAW || p->objective == OBJ_SQUAREDLOGERROR || p->objective == OBJ_PSEUDOHUBER;
    if (reg_loss && y == 1.0f) w *= p->scale_pos_weight;
    float pr = margins[r], g, h;
    if (p->objective == OBJ_SQUAREDERROR) { g = pr - y; h = 1.0f; }
    else if (p->objective == OBJ_SQUAREDLOGERROR) {
      if (!(y > -1.0f)) err = -3;
      pr = fmaxf(pr, -1.0f + 1e-6f);
      g = (log1pf(pr) - log1pf(y)) / (pr + 1.0f);
      h = fmaxf((-log1pf(pr) + log1pf(y) + 1.0f) / ((pr + 1.0f) * (pr + 1.0f)), 1e-6f);
    } else if (p->objective == OBJ_PSEUDOHUBER) {
      const float z = pr - y, s2 = p->huber_slope * p->huber_slope, scale_sqrt = sqrtf(1.0f + z * z / s2);
      g = z / scale_sqrt; h = s2 / ((s2 + z * z) * scale_sqrt);
    } else if (p->objective == OBJ_POISSON) {
      if (y < 0.0f) err = -4;
      g = expf(pr) - y; h = expf(pr + p->poisson_max_delta_step);
    } else if (p->objective == OBJ_GAMMA) {
      if (!(y > 0.0f)) err = -5;
      const float ep = expf(pr);
      g = 1.0f - y / ep; h = y / ep;
    } else if (p->objective == OBJ_TWEEDIE) {
      if (y < 0.0f) err = -6;
      const float rho = p->tweedie_variance_power, e1 = expf((1.0f - rho) * pr), e2 = expf((2.0f - rho) * pr);
      g = -y * e1 + e2; h = -y * (1.0f - rho) * e1 + (2.0f - rho) * e2;
    } else if (p->objective == OBJ_HINGE) {
      const float yy = y * 2.0f - 1.0f;
      if (pr * yy < 1.0f) { g = -yy; h = 1.0f; } else { g = 0.0f; h = 1.17549435e-38f; }
    } else {
      if (y < 0.0f || y > 1.0f) err = -1;
      pr = orc_sigmoid(pr);
      g = pr - y;
      h = fmaxf(pr * (1.0f - pr), 1e-16f);
    }
    gpair[r * 2 + 0] = g * w;
    gpair[r * 2 + 1] = h * w;
  }
  return err;
}

/* Base score: one Newton stump at margin 0, then PredTransform.
 * [UPSTREAM src/objective/init_estimation.cc, src/tree/fit_stump.cc]
 * Returns the base_score in OUTPUT space (what the model file stores). */
float orc_base_score(const OrcParams* p, const float* labels, const float* weights, int64_t n) {
  if (p->objective == OBJ_SOFTPROB || p->objective == OBJ_SOFTMAX) return 0.5f;
  /* only the RegLossObj family fits an intercept in 3.0.x [UPSTREAM-RECALL]; the log-link objectives and hinge keep 0.5 */
  if (p->objective == OBJ_POISSON || p->objective == OBJ_GAMMA || p->objective == OBJ_TWEEDIE || p->objective == OBJ_HINGE) return 0.5f;
  if (n == 0) return 0.5f;
  float* zero = (float*)calloc((size_t)n, sizeof(float));
  float* gp = (float*)malloc(sizeof(float) * 2 * (size_t)n);
  orc_gradient(p, zero, labels, weights, n, gp);
  double G = 0, H = 0;
  for (int64_t r = 0; r < n; ++r) { G += gp[2 * r]; H += gp[2 * r + 1]; }
  free(zero); free(gp);
  float wgt = H <= 0.0 ? 0.0f : (float)(-G / H);
  /* logitraw too: base_score lives in probability space for every logistic objective, so that orc_prob_to_margin's logit
   * gives back the stump weight (storing the raw margin and taking its logit is NaN whenever mean(y) < 0.5) */
  if (p->objective == OBJ_BINARY_LOGISTIC || p->objective == OBJ_REG_LOGISTIC || p->objective == OBJ_LOGITRAW) return orc_sigmoid(wgt);
  return wgt;   /* squarederror: identity transform */
}

float orc_prob_to_margin(const OrcParams* p, float base_score) {
  if (p->objective == OBJ_BINARY_LOGISTIC || p->objective == OBJ_REG_LOGISTIC || p->objective == OBJ_LOGITRAW)
    return -logf(1.0f / base_score - 1.0f);
  if (p->objective == OBJ_POISSON || p->objective == OBJ_GAMMA || p->objective == OBJ_TWEEDIE) return logf(base_score);
  return base_score;
}

/* ------------------------------------------------------------------------------------------ */
/* Split arithmetic.  [UPSTREAM src/tree/param.h, src/tree/split_evaluator.h]                   */
/* ------------------------------------------------------------------------------------------ */
static inline double threshold_l1(double w, double alpha) {
  if (w > +alpha) return w - alpha;
  if (w < -alpha) return w + alpha;
  return 0.0;
}
static inline float calc_weight(const OrcParams* p, double G, double H) {
  if (H < p->min_child_weight || H <= 0.0) return 0.0f;
  double dw = -threshold_l1(G, p->alpha) / (H + p->lambda);
  if (p->max_delta_step != 0.0f && fabs(dw) > p->max_delta_step) dw = copysign((double)p->max_delta_step, dw);
  return (float)dw;
}
static inline float calc_gain_given_weight(const OrcParams* p, double G, double H, float w) {
  if (H <= 0.0) return 0.0f;
  if (p->max_delta_step == 0.0f) {
    double t = threshold_l1(G, p->alpha);
    return (float)(t * t / (H + p->lambda));
  }
  /* tree::CalcGainGivenWeight<ParamT, float>: -(2 G w + (H + lambda) w^2), evaluated in float */
  float g = (float)G, h = (float)H;
  return -(2.0f * g * w + (h + p->lambda) * w * w);
}
static inline float calc_gain(const OrcParams* p, double G, double H) {
  return calc_gain_given_weight(p, G, H, calc_weight(p, G, H));
}
static inline float calc_split_gain(const OrcParams* p, double GL, double HL, double GR, double HR);
/* exported for tests/test_oracle_fixture.py: the reference-held model fixture's node statistics are fed to exactly the
 * functions the trainer uses */
float orc_calc_weight(const OrcParams* p, double G, double H) { return calc_weight(p, G, H); }
float orc_calc_gain(const OrcParams* p, double G, double H) { return calc_gain(p, G, H); }
float orc_calc_split_gain(const OrcParams* p, double GL, double HL, double GR, double HR) { return calc_split_gain(p, GL, HL, GR, HR); }
static inline float calc_split_gain(const OrcParams* p, double GL, double HL, double GR, double HR) {
  float wl = calc_weight(p, GL, HL), wr = calc_weight(p, GR, HR);
  return calc_gain_given_weight(p, GL, HL, wl) + calc_gain_given_weight(p, GR, HR, wr);
}

typedef struct {
  float loss_chg; int32_t findex; float split_value; int32_t split_bin; int32_t default_left;
  double GL, HL, GR, HR;
} Split;

/* [UPSTREAM src/tree/param.h SplitEntry::NeedReplace / Update]: larger loss_chg wins; a tie keeps
 * the LOWER feature index; within one feature the first candidate in scan order wins (strict >). */
static inline int need_replace(float cur_loss, int cur_idx, float new_loss, int new_idx) {
  if (isinf(new_loss)) return 0;
  if (cur_idx <= new_idx) return new_loss > cur_loss;
  return !(cur_loss > new_loss);
}
static inline void split_update(Split* best, float loss_chg, int f, float value, int bin, int dleft,
                                double GL, double HL, double GR, double HR) {
  if (need_replace(best->loss_chg, best->findex, loss_chg, f)) {
    best->loss_chg = loss_chg; best->findex = f; best->split_value = value; best->split_bin = bin;
    best->default_left = dleft; best->GL = GL; best->HL = HL; best->GR = GR; best->HR = HR;
  }
}

/* Monotone constraints.  [UPSTREAM src/tree/split_evaluator.h TreeEvaluator::SplitEvaluator: CalcWeight clamps to the node's
 * [lower, upper]; CalcGainGivenWeight takes the general form -(2 G w + (H + lambda) w^2) whenever constraints exist;
 * CalcSplitGain returns -inf when the child weights violate the feature's constraint; AddSplit hands mid = (wl + wr) / 2 down
 * as the children's new bound on the constrained side] */
typedef struct { const int32_t* c; float lo, hi; } Mono;      /* c == NULL: unconstrained */
static inline float clamp_w(float w, float lo, float hi) { return w < lo ? lo : (w > hi ? hi : w); }
static inline float gain_at_weight(const OrcParams* p, double G, double H, float w) {
  if (H <= 0.0) return 0.0f;
  const float g = (float)G, h = (float)H;
  return -(2.0f * g * w + (h + p->lambda) * w * w);
}
static inline float split_loss_chg(const OrcParams* p, const Mono* mn, int f, double GL, double HL, double GR, double HR, float root_gain) {
  if (!mn || !mn->c) return (float)(calc_split_gain(p, GL, HL, GR, HR) - root_gain);
  const float wl = clamp_w(calc_weight(p, GL, HL), mn->lo, mn->hi), wr = clamp_w(calc_weight(p, GR, HR), mn->lo, mn->hi);
  const int cf = mn->c[f];
  if (cf != 0 && !(cf > 0 ? wl <= wr : wl >= wr)) return -INFINITY;
  return gain_at_weight(p, GL, HL, wl) + gain_at_weight(p, GR, HR, wr) - root_gain;
}

/* hist: total_bins x 2 doubles (g,h) for one node. feat_mask: F bytes (1 = usable) or NULL.
 * [UPSTREAM src/tree/hist/evaluate_splits.h EnumerateSplit<+1/-1>, EvaluateSplits] */
static void eval_split_mono(const OrcParams* p, const double* hist, const int32_t* cut_ptrs, const float* cut_vals,
                    const float* min_vals, int32_t F, const uint8_t* feat_mask, double G, double H,
                    float root_gain, const Mono* mn, Split* out) {
  Split best; memset(&best, 0, sizeof best); best.split_bin = -1;     /* SplitEntry{}: loss_chg 0, sindex 0 */
  for (int f = 0; f < F; ++f) {
    if (feat_mask && !feat_mask[f]) continue;
    int ib = cut_ptrs[f], ie = cut_ptrs[f + 1];
    Split fb; memset(&fb, 0, sizeof fb); fb.split_bin = -1;
    double GL = 0, HL = 0;
    for (int i = ib; i < ie; ++i) {           /* forward: missing goes right, threshold = cut[i] */
      GL += hist[2 * i]; HL += hist[2 * i + 1];
      double GR = G - GL, HR = H - HL;
      if (HL >= p->min_child_weight && HR >= p->min_child_weight) {
        float lc = split_loss_chg(p, mn, f, GL, HL, GR, HR, root_gain);
        split_update(&fb, lc, f, cut_vals[i], i - ib, 0, GL, HL, GR, HR);
      }
    }
    if (!(GL == G && HL == H)) {              /* SplitContainsMissingValues: backward scan, missing goes left */
      double GRr = 0, HRr = 0;
      for (int i = ie - 1; i >= ib; --i) {
        GRr += hist[2 * i]; HRr += hist[2 * i + 1];
        double GLl = G - GRr, HLl = H - HRr;
        if (HRr >= p->min_child_weight && HLl >= p->min_child_weight) {
          float lc = split_loss_chg(p, mn, f, GLl, HLl, GRr, HRr, root_gain);
          float sv = (i == ib) ? min_vals[f] : cut_vals[i - 1];
          split_update(&fb, lc, f, sv, i - ib - 1, 1, GLl, HLl, GRr, HRr);
        }
      }
    }
    if (need_replace(best.loss_chg, best.findex, fb.loss_chg, fb.findex)) best = fb;
  }
  *out = best;
}

void orc_eval_split(const OrcParams* p, const double* hist, const int32_t* cut_ptrs, const float* cut_vals,
                    const float* min_vals, int32_t F, const uint8_t* feat_mask, double G, double H,
                    float root_gain, Split* out) {
  eval_split_mono(p, hist, cut_ptrs, cut_vals, min_vals, F, feat_mask, G, H, root_gain, NULL, out);
}

/* ------------------------------------------------------------------------------------------ */
/* Histogram build.  [UPSTREAM src/common/hist_util.cc BuildHist, src/tree/hist/histogram.h]    */
/* bins: n x F row-major (global bin = cut_ptrs[f] + bins[r,f]); gpair: (g,h) floats, stride    */
/* gstride floats between rows (2 for K=1).  rows: row ids (NULL = 0..nrows-1).                 */
/* ------------------------------------------------------------------------------------------ */
void orc_build_hist(const uint8_t* bins, int32_t F, const int32_t* cut_ptrs, const float* gpair,
                    int64_t gstride, const uint32_t* rows, int64_t nrows, int32_t has_missing,
                    double* hist /* total_bins*2 */) {
  const int total_bins = cut_ptrs[F];
  memset(hist, 0, sizeof(double) * 2 * (size_t)total_bins);
  int nt = 1;
#ifdef _OPENMP
  nt = omp_get_max_threads();
#endif
  /* one private histogram per thread costs a zero + reduce of 16 B x total_bins: only use as many threads as the
   * balance row work (nrows x F / nt) against that overhead (nt x total_bins): nt ~ sqrt(nrows F / (2 total_bins)) */
  { double want = sqrt((double)nrows * (double)F / (2.0 * (double)(total_bins > 0 ? total_bins : 1))); if (want < 1.0) want = 1.0; if (want < (double)nt) nt = (int)want; }
  static double* g_priv = NULL; static size_t g_priv_cap = 0;
  double* priv = NULL;
  if (nt > 1) {
    size_t need = (size_t)nt * 2 * total_bins;
    if (need > g_priv_cap) { free(g_priv); g_priv = (double*)malloc(sizeof(double) * need); g_priv_cap = need; }
    priv = g_priv;
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int t = 0; t < nt; ++t) memset(priv + (size_t)t * 2 * total_bins, 0, sizeof(double) * 2 * (size_t)total_bins);
  }
#pragma omp parallel num_threads(nt)
  {
    int tid = 0;
#ifdef _OPENMP
    tid = omp_get_thread_num();
#endif
    double* h = nt > 1 ? priv + (size_t)tid * 2 * total_bins : hist;
#pragma omp for schedule(static)
    for (int64_t i = 0; i < nrows; ++i) {
      int64_t r = rows ? rows[i] : i;
      const uint8_t* b = bins + r * F;
      double g = gpair[r * gstride], hh = gpair[r * gstride + 1];
      for (int f = 0; f < F; ++f) {
        if (has_missing && b[f] == ORC_MISSING_BIN) continue;
        int idx = cut_ptrs[f] + b[f];
        h[2 * idx] += g; h[2 * idx + 1] += hh;
      }
    }
  }
  if (nt > 1) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < 2 * total_bins; ++i) {
      double s = 0; for (int t = 0; t < nt; ++t) s += priv[(size_t)t * 2 * total_bins + i];
      hist[i] = s;
    }
  }
}

/* Fixed-point mirror of the product's integer histogram: gq,hq are the int32 quantised gradients,
 * accumulation is exact int64. Layout out: F x 256 x 2 (g,h).  Used for bit-exact kernel tests. */
void orc_build_hist_fixed(const uint8_t* bins, int32_t F, const int32_t* gq, const int32_t* hq,
                          const uint32_t* rows, int64_t nrows, int64_t* hist /* F*256*2 */) {
  memset(hist, 0, sizeof(int64_t) * 2 * 256 * (size_t)F);
  for (int64_t i = 0; i < nrows; ++i) {
    int64_t r = rows ? rows[i] : i;
    const uint8_t* b = bins + r * F;
    for (int f = 0; f < F; ++f) {
      int64_t idx = ((int64_t)f * 256 + b[f]) * 2;
      hist[idx] += gq[r]; hist[idx + 1] += hq[r];
    }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* Model: flat arrays, trees concatenated.                                                     */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_trees, cap_trees;
  int64_t n_nodes, cap_nodes;
  int64_t* tree_offset;    /* n_trees+1 */
  int32_t* tree_info;      /* class id per tree */
  int32_t *left, *right, *parent, *split_index, *split_bin;
  uint8_t* default_left;
  float *split_cond, *base_weight, *loss_chg, *sum_hess;
} OrcModel;

static void model_reserve_nodes(OrcModel* m, int64_t extra) {
  if (m->n_nodes + extra <= m->cap_nodes) return;
  int64_t cap = m->cap_nodes ? m->cap_nodes * 2 : 1024;
  while (cap < m->n_nodes + extra) cap *= 2;
#define RE(ptr, T) m->ptr = (T*)realloc(m->ptr, sizeof(T) * (size_t)cap)
  RE(left, int32_t); RE(right, int32_t); RE(parent, int32_t); RE(split_index, int32_t); RE(split_bin, int32_t);
  RE(default_left, uint8_t); RE(split_cond, float); RE(base_weight, float); RE(loss_chg, float); RE(sum_hess, float);
#undef RE
  m->cap_nodes = cap;
}
static void model_reserve_trees(OrcModel* m) {
  if (m->n_trees + 1 <= m->cap_trees) return;
  int cap = m->cap_trees ? m->cap_trees * 2 : 64;
  m->tree_offset = (int64_t*)realloc(m->tree_offset, sizeof(int64_t) * (size_t)(cap + 1));
  m->tree_info = (int32_t*)realloc(m->tree_info, sizeof(int32_t) * (size_t)cap);
  if (m->cap_trees == 0) m->tree_offset[0] = 0;
  m->cap_trees = cap;
}

/* ------------------------------------------------------------------------------------------ */
/* Trainer state                                                                               */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  OrcParams p;
  int64_t n; int32_t F;
  const uint8_t* bins;        /* borrowed, n x F */
  const int32_t* cut_ptrs; const float* cut_vals; const float* min_vals;   /* borrowed */
  const float* labels; const float* weights;                               /* borrowed */
  int has_missing;
  float base_score;           /* output space */
  float* margins;             /* n x K */
  float* gpair;               /* n x K x 2 */
  uint32_t* ridx; uint32_t* ridx_tmp;     /* row-id partition buffers */
  int32_t* row_leaf;          /* leaf node (tree-local id) per row of the tree being grown */
  OrcModel model;
  int32_t iter;               /* boosted rounds so far */
  int32_t* monotone;          /* F entries (-1, 0, +1) or NULL */
  uint8_t* ic_sets; int32_t n_ic_sets;    /* interaction constraints: membership matrix [n_ic_sets][F], or NULL */
  int32_t quant_bits;         /* 0 = reference behaviour; >0 = study knob: round gpair to a 2^-k grid like the
                                 product's fixed-point histogram (scale = power of two from max|g|, max h) */
} OrcTrainer;

/* counter-based RNG shared with the product (csrc/rng.h): splitmix64 on (seed, stream, index) */
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ULL; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL; return x ^ (x >> 31);
}
static inline float rng_uniform(uint32_t seed, uint64_t stream, uint64_t idx) {
  uint64_t h = splitmix64(splitmix64(((uint64_t)seed << 32) ^ stream) ^ idx);
  return (float)(h >> 40) * (1.0f / 16777216.0f);
}

OrcTrainer* orc_trainer_create(const OrcParams* p, const uint8_t* bins, int64_t n, int32_t F,
                               const int32_t* cut_ptrs, const float* cut_vals, const float* min_vals,
                               const float* labels, const float* weights, int32_t has_missing,
                               float base_score, int32_t base_score_set) {
  OrcTrainer* t = (OrcTrainer*)calloc(1, sizeof(OrcTrainer));
  t->p = *p; t->n = n; t->F = F; t->bins = bins; t->cut_ptrs = cut_ptrs; t->cut_vals = cut_vals;
  t->min_vals = min_vals; t->labels = labels; t->weights = weights; t->has_missing = has_missing;
  const int K = p->num_class > 1 ? p->num_class : 1;
#ifdef _OPENMP
  if (p->nthread > 0) omp_set_num_threads(p->nthread);
#endif
  t->base_score = base_score_set ? base_score : orc_base_score(p, labels, weights, n);
  float bm = orc_prob_to_margin(p, t->base_score);
  t->margins = (float*)malloc(sizeof(float) * (size_t)(n * K > 0 ? n * K : 1));
  for (int64_t i = 0; i < n * K; ++i) t->margins[i] = bm;
  t->gpair = (float*)malloc(sizeof(float) * 2 * (size_t)(n * K > 0 ? n * K : 1));
  t->ridx = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(n > 0 ? n : 1));
  t->ridx_tmp = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(n > 0 ? n : 1));
  t->row_leaf = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
  return t;
}

void orc_trainer_free(OrcTrainer* t) {
  if (!t) return;
  free(t->margins); free(t->gpair); free(t->ridx); free(t->ridx_tmp); free(t->row_leaf); free(t->monotone); free(t->ic_sets);
  OrcModel* m = &t->model;
  free(m->tree_offset); free(m->tree_info); free(m->left); free(m->right); free(m->parent);
  free(m->split_index); free(m->split_bin); free(m->default_left); free(m->split_cond);
  free(m->base_weight); free(m->loss_chg); free(m->sum_hess);
  free(t);
}

typedef struct {
  int nid, depth; Split split; double G, H; float root_gain, weight;
  float lo, hi;            /* weight interval of the node under monotone constraints */
  uint8_t* path; uint8_t* allowed;   /* interaction constraints: features on the path / features this node may split on (owned, F bytes) */
  int64_t begin, count;    /* row segment in ridx */
  double* hist;            /* owned */
} Cand;

/* [UPSTREAM-RECALL src/tree/constraints.cc FeatureInteractionConstraintHost]: the root may use any feature; a child may use the
 * features on its path plus every feature of each constraint set that contains ALL path features. */
void orc_set_interaction(OrcTrainer* t, const uint8_t* sets, int32_t n_sets) {
  free(t->ic_sets); t->ic_sets = NULL; t->n_ic_sets = 0;
  if (n_sets <= 0) return;
  t->ic_sets = (uint8_t*)malloc((size_t)n_sets * (size_t)t->F); memcpy(t->ic_sets, sets, (size_t)n_sets * (size_t)t->F); t->n_ic_sets = n_sets;
}
static void cand_free(Cand* c) { free(c->hist); c->hist = NULL; free(c->path); c->path = NULL; free(c->allowed); c->allowed = NULL; }
static void interaction_child(const OrcTrainer* t, const uint8_t* parent_path, int f, uint8_t** path_out, uint8_t** allowed_out) {
  const int F = t->F;
  uint8_t* path = (uint8_t*)malloc((size_t)F); uint8_t* allowed = (uint8_t*)malloc((size_t)F);
  for (int j = 0; j < F; ++j) { path[j] = (parent_path[j] || j == f) ? 1 : 0; allowed[j] = path[j]; }
  for (int s = 0; s < t->n_ic_sets; ++s) {
    const uint8_t* set = t->ic_sets + (size_t)s * F;
    int relevant = 1;
    for (int j = 0; j < F && relevant; ++j) if (path[j] && !set[j]) relevant = 0;
    if (relevant) for (int j = 0; j < F; ++j) if (set[j]) allowed[j] = 1;
  }
  *path_out = path; *allowed_out = allowed;
}
/* usable features of a node = sampling mask AND interaction-allowed mask (either may be absent) */
static const uint8_t* combine_masks(const uint8_t* a, const uint8_t* b, int F, uint8_t* scratch) {
  if (!a) return b;
  if (!b) return a;
  for (int j = 0; j < F; ++j) scratch[j] = a[j] && b[j];
  return scratch;
}

static int new_node(OrcModel* m, int64_t base, int parent) {
  model_reserve_nodes(m, 1);
  int64_t i = m->n_nodes++;
  m->left[i] = -1; m->right[i] = -1; m->parent[i] = parent; m->split_index[i] = 0; m->split_bin[i] = -1;
  m->default_left[i] = 0; m->split_cond[i] = 0; m->base_weight[i] = 0; m->loss_chg[i] = 0; m->sum_hess[i] = 0;
  return (int)(i - base);
}

/* Grow one tree on gradient column k.  [UPSTREAM src/tree/updater_quantile_hist.cc, src/tree/driver.h,
 * src/tree/hist/histogram.h (subtraction trick, build the child with the smaller hessian sum),
 * src/common/partition_builder.h (stable partition, bin <= split_bin -> left)] */
/* child[f] = parent[f] && fewer than keep = max(1, floor(frac * |parent|)) parent features have a smaller hash (ties: lower index) */
static void subset_mask(const uint8_t* parent, int F, float frac, uint32_t seed, uint64_t stream, uint8_t* child) {
  if (frac >= 1.0f) { memcpy(child, parent, (size_t)F); return; }
  int cnt = 0; for (int f = 0; f < F; ++f) cnt += parent[f] ? 1 : 0;
  int keep = (int)floorf(frac * (float)cnt); if (keep < 1) keep = 1;
  for (int f = 0; f < F; ++f) {
    child[f] = 0;
    if (!parent[f]) continue;
    float u = rng_uniform(seed, stream, (uint64_t)f);
    int rank = 0;
    for (int g = 0; g < F; ++g) {
      if (!parent[g]) continue;
      float v = rng_uniform(seed, stream, (uint64_t)g);
      if (v < u || (v == u && g < f)) ++rank;
    }
    child[f] = rank < keep;
  }
}

/* Stable partition of the row segment [begin, begin + count) by the split (feature f, bin sb, default direction dl):
 * lefts first, rights after, both in their original order.  [UPSTREAM src/common/partition_builder.h]  Parallel over
 * row blocks (count, prefix, scatter), so that the CPU baseline scales with the host's cores like upstream's does. */
static void partition_segment(OrcTrainer* t, int64_t begin, int64_t count, int f, int sb, int dl, int64_t* nl_out) {
  const int F = t->F;
  uint32_t* seg = t->ridx + begin; uint32_t* tmp = t->ridx_tmp;
  int nt = 1;
#ifdef _OPENMP
  nt = omp_get_max_threads();
#endif
  if (count < 262144) nt = 1; else if ((int64_t)nt > count / 65536) nt = (int)(count / 65536);
  if (nt <= 1) {
    int64_t nl = 0, nr = 0;
    for (int64_t i = 0; i < count; ++i) {
      uint32_t r = seg[i]; uint8_t b = t->bins[(int64_t)r * F + f];
      int go_left = (t->has_missing && b == ORC_MISSING_BIN) ? dl : ((int)b <= sb);
      if (go_left) seg[nl++] = r; else tmp[nr++] = r;
    }
    memcpy(seg + nl, tmp, sizeof(uint32_t) * (size_t)nr);
    *nl_out = nl; return;
  }
  int64_t* cntl = (int64_t*)calloc((size_t)nt + 1, sizeof(int64_t));
  const int64_t blk = (count + nt - 1) / nt;
#pragma omp parallel for schedule(static, 1) num_threads(nt)
  for (int th = 0; th < nt; ++th) {
    int64_t i0 = th * blk, i1 = i0 + blk < count ? i0 + blk : count, c = 0;
    for (int64_t i = i0; i < i1; ++i) {
      uint8_t b = t->bins[(int64_t)seg[i] * F + f];
      c += (t->has_missing && b == ORC_MISSING_BIN) ? dl : ((int)b <= sb);
    }
    cntl[th + 1] = c;
  }
  for (int th = 0; th < nt; ++th) cntl[th + 1] += cntl[th];
  const int64_t nl = cntl[nt];
#pragma omp parallel for schedule(static, 1) num_threads(nt)
  for (int th = 0; th < nt; ++th) {
    int64_t i0 = th * blk, i1 = i0 + blk < count ? i0 + blk : count;
    int64_t ol = cntl[th], orr = nl + (i0 - cntl[th]);
    for (int64_t i = i0; i < i1; ++i) {
      uint32_t r = seg[i]; uint8_t b = t->bins[(int64_t)r * F + f];
      int go_left = (t->has_missing && b == ORC_MISSING_BIN) ? dl : ((int)b <= sb);
      if (go_left) tmp[ol++] = r; else tmp[orr++] = r;
    }
  }
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int64_t i = 0; i < count; ++i) seg[i] = tmp[i];
  free(cntl);
  *nl_out = nl;
}

static void grow_tree(OrcTrainer* t, int k, int tree_index) {
  const OrcParams* p = &t->p;
  const int K = p->num_class > 1 ? p->num_class : 1;
  const int F = t->F; const int64_t n = t->n;
  const int total_bins = t->cut_ptrs[F];
  OrcModel* m = &t->model;
  model_reserve_trees(m);
  const int64_t base = m->n_nodes;
  const float* gp = t->gpair + 2 * k; const int64_t gs = 2 * K;

  /* column sampling [UPSTREAM src/common/random.h ColumnSampler: bytree, bylevel inside it, bynode inside that; a subset keeps
   * max(1, floor(frac * |parent|)) features].  Upstream shuffles with a mt19937 (not restatable): oracle and product keep the
   * features of the parent set with the smallest counter-based hash instead (subset_mask). */
  const int sampling = p->colsample_bytree < 1.0f || p->colsample_bylevel < 1.0f || p->colsample_bynode < 1.0f;
  uint8_t* tree_mask = NULL; uint8_t* level_masks = NULL; uint8_t* node_mask = NULL;
  const int maxd = p->max_depth > 0 ? p->max_depth : 1;
  uint8_t* ic_scratch = (uint8_t*)malloc((size_t)(F > 0 ? F : 1));
  if (sampling) {
    uint8_t* all = (uint8_t*)malloc((size_t)F); memset(all, 1, (size_t)F);
    tree_mask = (uint8_t*)malloc((size_t)F);
    subset_mask(all, F, p->colsample_bytree, p->seed, 0x1000ull + (uint64_t)tree_index, tree_mask);
    level_masks = (uint8_t*)malloc((size_t)F * (size_t)maxd);
    for (int d = 0; d < maxd; ++d)
      subset_mask(tree_mask, F, p->colsample_bylevel, p->seed, 0x300000ull + 64ull * (uint64_t)tree_index + (uint64_t)d, level_masks + (size_t)d * F);
    node_mask = (uint8_t*)malloc((size_t)F);
    free(all);
  }
#define NODE_MASK(depth, nid) (!sampling ? NULL : (subset_mask(level_masks + (size_t)((depth) < maxd ? (depth) : maxd - 1) * F, F, p->colsample_bynode, p->seed, \
                               0x80000000ull + ((uint64_t)tree_index << 20) + (uint64_t)(nid), node_mask), node_mask))

  for (int64_t r = 0; r < n; ++r) t->ridx[r] = (uint32_t)r;
  Cand* cur = (Cand*)calloc(1, sizeof(Cand)); int ncur = 0;
  /* root */
  {
    Cand c; memset(&c, 0, sizeof c);
    c.nid = new_node(m, base, 2147483647); c.depth = 0; c.begin = 0; c.count = n;
    c.hist = (double*)malloc(sizeof(double) * 2 * (size_t)total_bins);
    orc_build_hist(t->bins, F, t->cut_ptrs, gp, gs, NULL, n, t->has_missing, c.hist);
    double G = 0, H = 0;
    if (!t->has_missing) { for (int i = t->cut_ptrs[0]; i < t->cut_ptrs[1]; ++i) { G += c.hist[2 * i]; H += c.hist[2 * i + 1]; } }
    else { for (int64_t r = 0; r < n; ++r) { G += gp[r * gs]; H += gp[r * gs + 1]; } }
    c.G = G; c.H = H; c.lo = -INFINITY; c.hi = INFINITY;
    if (t->ic_sets) { c.path = (uint8_t*)calloc((size_t)F, 1); c.allowed = (uint8_t*)malloc((size_t)F); memset(c.allowed, 1, (size_t)F); }
    c.weight = calc_weight(p, G, H);
    c.root_gain = t->monotone ? gain_at_weight(p, G, H, c.weight) : calc_gain(p, G, H);
    m->base_weight[base] = c.weight; m->sum_hess[base] = (float)H; m->split_cond[base] = p->eta * c.weight;
    { Mono mn = { t->monotone, c.lo, c.hi }; eval_split_mono(p, c.hist, t->cut_ptrs, t->cut_vals, t->min_vals, F, combine_masks(NODE_MASK(0, 0), c.allowed, F, ic_scratch), G, H, c.root_gain, &mn, &c.split); }
    cur[0] = c; ncur = 1;
  }
  int num_leaves = 1;
  /* One Driver::Pop batch: depthwise = every open candidate of the current depth in increasing nid; lossguide = the single best
   * open candidate (max loss_chg, ties to the smaller nid), and an invalid top entry ends the tree (upstream Driver::Pop returns
   * an empty batch).  [UPSTREAM src/tree/driver.h, src/tree/hist/expand_entry.h] */
  const int lossguide = p->grow_policy == 1;
  while (ncur > 0) {
    Cand* next = (Cand*)calloc((size_t)ncur * 2 + 2, sizeof(Cand)); int nnext = 0;
    int stop = 0;
    int first = 0, last = ncur;
    if (lossguide) {
      int bi = 0;
      for (int ci = 1; ci < ncur; ++ci)
        if (cur[ci].split.loss_chg > cur[bi].split.loss_chg || (cur[ci].split.loss_chg == cur[bi].split.loss_chg && cur[ci].nid < cur[bi].nid)) bi = ci;
      for (int ci = 0; ci < ncur; ++ci) if (ci != bi) next[nnext++] = cur[ci];     /* everything else stays open */
      Cand tmp = cur[bi]; cur[bi] = cur[0]; cur[0] = tmp;
      first = 0; last = 1;
    }
    for (int ci = first; ci < last; ++ci) {
      Cand* c = &cur[ci];
      int valid = 1;
      if (!(c->split.loss_chg > K_RT_EPS)) valid = 0;
      else if (c->split.HL == 0 || c->split.HR == 0) valid = 0;
      else if (c->split.loss_chg < p->gamma) valid = 0;
      else if (p->max_depth > 0 && c->depth == p->max_depth) valid = 0;
      else if (p->max_leaves > 0 && num_leaves == p->max_leaves) valid = 0;
      if (!valid) { cand_free(c); if (lossguide) stop = 1; continue; }
      num_leaves++;
      /* ApplySplit / ExpandNode */
      int64_t gi = base + c->nid;
      int L = new_node(m, base, c->nid), R = new_node(m, base, c->nid);
      gi = base + c->nid;
      float wl = calc_weight(p, c->split.GL, c->split.HL), wr = calc_weight(p, c->split.GR, c->split.HR);
      float llo = c->lo, lhi = c->hi, rlo = c->lo, rhi = c->hi;
      if (t->monotone) {            /* children weights clamped by the PARENT's interval; AddSplit */
        wl = clamp_w(wl, c->lo, c->hi); wr = clamp_w(wr, c->lo, c->hi);
        const float mid = (wl + wr) / 2.0f; const int cf = t->monotone[c->split.findex];
        if (cf < 0) { llo = mid; rhi = mid; } else if (cf > 0) { lhi = mid; rlo = mid; }
      }
      m->left[gi] = L; m->right[gi] = R; m->split_index[gi] = c->split.findex; m->split_cond[gi] = c->split.split_value;
      m->split_bin[gi] = c->split.split_bin; m->default_left[gi] = (uint8_t)c->split.default_left;
      m->base_weight[gi] = c->weight; m->loss_chg[gi] = c->split.loss_chg; m->sum_hess[gi] = (float)c->H;
      m->split_cond[base + L] = p->eta * wl; m->base_weight[base + L] = p->eta * wl; m->sum_hess[base + L] = (float)c->split.HL;
      m->split_cond[base + R] = p->eta * wr; m->base_weight[base + R] = p->eta * wr; m->sum_hess[base + R] = (float)c->split.HR;
      /* stable partition of the node's row segment */
      int f = c->split.findex, sb = c->split.split_bin, dl = c->split.default_left;
      int64_t nl = 0, nr = 0;
      partition_segment(t, c->begin, c->count, f, sb, dl, &nl);
      nr = c->count - nl;
      /* children candidates */
      int child_ok = 1;
      if (p->max_depth > 0 && c->depth + 1 >= p->max_depth) child_ok = 0;
      if (p->max_leaves > 0 && num_leaves >= p->max_leaves) child_ok = 0;
      Cand cl, cr; memset(&cl, 0, sizeof cl); memset(&cr, 0, sizeof cr);
      cl.nid = L; cr.nid = R; cl.depth = cr.depth = c->depth + 1;
      cl.begin = c->begin; cl.count = nl; cr.begin = c->begin + nl; cr.count = nr;
      cl.G = c->split.GL; cl.H = c->split.HL; cr.G = c->split.GR; cr.H = c->split.HR;
      cl.lo = llo; cl.hi = lhi; cr.lo = rlo; cr.hi = rhi;
      if (t->ic_sets) { interaction_child(t, c->path, c->split.findex, &cl.path, &cl.allowed); interaction_child(t, c->path, c->split.findex, &cr.path, &cr.allowed); }
      if (child_ok) {
        int fewer_right = c->split.HR < c->split.HL;
        Cand* bld = fewer_right ? &cr : &cl; Cand* sub = fewer_right ? &cl : &cr;
        bld->hist = (double*)malloc(sizeof(double) * 2 * (size_t)total_bins);
        orc_build_hist(t->bins, F, t->cut_ptrs, gp, gs, t->ridx + bld->begin, bld->count, t->has_missing, bld->hist);
        sub->hist = c->hist; c->hist = NULL;
        for (int i = 0; i < 2 * total_bins; ++i) sub->hist[i] -= bld->hist[i];
        Cand* two[2] = { &cl, &cr };
        for (int s = 0; s < 2; ++s) {
          Cand* ch = two[s];
          ch->weight = t->monotone ? clamp_w(calc_weight(p, ch->G, ch->H), ch->lo, ch->hi) : calc_weight(p, ch->G, ch->H);
          ch->root_gain = t->monotone ? gain_at_weight(p, ch->G, ch->H, ch->weight) : calc_gain(p, ch->G, ch->H);
          { Mono mn = { t->monotone, ch->lo, ch->hi }; eval_split_mono(p, ch->hist, t->cut_ptrs, t->cut_vals, t->min_vals, F, combine_masks(NODE_MASK(ch->depth, ch->nid), ch->allowed, F, ic_scratch), ch->G, ch->H, ch->root_gain, &mn, &ch->split); }
          if (ch->split.loss_chg > K_RT_EPS) next[nnext++] = *ch; else cand_free(ch);
        }
      } else { cand_free(&cl); cand_free(&cr); }
      cand_free(c);
    }
    free(cur); cur = next; ncur = nnext;
    if (stop) { for (int ci = 0; ci < ncur; ++ci) cand_free(&cur[ci]); ncur = 0; }
  }
  free(cur);
  free(tree_mask); free(level_masks); free(node_mask); free(ic_scratch);
#undef NODE_MASK
  /* finalize tree + prediction cache: traverse by bins (exact for training rows) */
  m->tree_offset[m->n_trees + 1] = m->n_nodes; m->tree_info[m->n_trees] = k; m->n_trees++;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n; ++r) {
    int nid = 0;
    while (m->left[base + nid] != -1) {
      int64_t gi = base + nid; int f = m->split_index[gi];
      uint8_t b = t->bins[r * F + f];
      int go_left = (t->has_missing && b == ORC_MISSING_BIN) ? m->default_left[gi] : ((int)b <= m->split_bin[gi]);
      nid = go_left ? m->left[gi] : m->right[gi];
    }
    t->row_leaf[r] = nid;
    t->margins[r * K + k] += m->split_cond[base + nid];
  }
}

/* One boosting round.  [UPSTREAM src/learner.cc UpdateOneIter, src/gbm/gbtree.cc DoBoost] */
int orc_update_one_iter(OrcTrainer* t) {
  const OrcParams* p = &t->p;
  const int K = p->num_class > 1 ? p->num_class : 1;
  int rc = orc_gradient(p, t->margins, t->labels, t->weights, t->n, t->gpair);
  if (rc) return rc;
  if (p->subsample < 1.0f) {   /* Bernoulli row mask: unsampled rows get a zero gradient pair */
    for (int64_t r = 0; r < t->n; ++r)
      if (!(rng_uniform(p->seed, 0x2000 + (uint64_t)t->iter, (uint64_t)r) < p->subsample))
        for (int k = 0; k < K; ++k) { t->gpair[(r * K + k) * 2] = 0; t->gpair[(r * K + k) * 2 + 1] = 0; }
  }
  if (t->quant_bits > 0) {
    float mg = 0, mh = 0;
    for (int64_t i = 0; i < t->n * K; ++i) { mg = fmaxf(mg, fabsf(t->gpair[2 * i])); mh = fmaxf(mh, t->gpair[2 * i + 1]); }
    int eg, eh; frexpf(mg, &eg); frexpf(mh, &eh);      /* m < 2^e */
    /* the product's scales_kernel with grad_bits = quant_bits - 1: |g_q| <= 2^grad_bits, h_q <= 2^(grad_bits + 1) */
    float sg = ldexpf(1.0f, t->quant_bits - 1 - eg), sh = ldexpf(1.0f, t->quant_bits - eh);
    for (int64_t i = 0; i < t->n * K; ++i) {
      t->gpair[2 * i] = rintf(t->gpair[2 * i] * sg) / sg;
      t->gpair[2 * i + 1] = rintf(t->gpair[2 * i + 1] * sh) / sh;
    }
  }
  for (int k = 0; k < K; ++k) grow_tree(t, k, t->iter * K + k);
  t->iter++;
  return 0;
}

/* accessors for the Python wrapper */
void orc_set_quant_bits(OrcTrainer* t, int32_t bits) { t->quant_bits = bits; }
void orc_set_monotone(OrcTrainer* t, const int32_t* c, int32_t ncon) {
  free(t->monotone); t->monotone = NULL;
  int any = 0; for (int i = 0; i < ncon; ++i) any |= c[i] != 0;
  if (!any) return;
  t->monotone = (int32_t*)calloc((size_t)t->F, sizeof(int32_t));
  for (int i = 0; i < ncon && i < t->F; ++i) t->monotone[i] = c[i];
}
void orc_set_margins(OrcTrainer* t, const float* m) { const int K = t->p.num_class > 1 ? t->p.num_class : 1; memcpy(t->margins, m, sizeof(float) * (size_t)(t->n * K)); }
int32_t orc_num_trees(const OrcTrainer* t) { return t->model.n_trees; }
int64_t orc_num_nodes(const OrcTrainer* t) { return t->model.n_nodes; }
float orc_get_base_score(const OrcTrainer* t) { return t->base_score; }
const float* orc_margins(const OrcTrainer* t) { return t->margins; }
const float* orc_gpair(const OrcTrainer* t) { return t->gpair; }
void orc_export_model(const OrcTrainer* t, int64_t* tree_offset, int32_t* tree_info, int32_t* left, int32_t* right,
                      int32_t* parent, int32_t* split_index, int32_t* split_bin, uint8_t* default_left,
                      float* split_cond, float* base_weight, float* loss_chg, float* sum_hess) {
  const OrcModel* m = &t->model;
  memcpy(tree_offset, m->tree_offset, sizeof(int64_t) * (size_t)(m->n_trees + 1));
  memcpy(tree_info, m->tree_info, sizeof(int32_t) * (size_t)m->n_trees);
  size_t nn = (size_t)m->n_nodes;
  memcpy(left, m->left, 4 * nn); memcpy(right, m->right, 4 * nn); memcpy(parent, m->parent, 4 * nn);
  memcpy(split_index, m->split_index, 4 * nn); memcpy(split_bin, m->split_bin, 4 * nn);
  memcpy(default_left, m->default_left, nn); memcpy(split_cond, m->split_cond, 4 * nn);
  memcpy(base_weight, m->base_weight, 4 * nn); memcpy(loss_chg, m->loss_chg, 4 * nn); memcpy(sum_hess, m->sum_hess, 4 * nn);
}

/* ------------------------------------------------------------------------------------------ */
/* Predictor.  [UPSTREAM src/predictor/cpu_predictor.cc; src/tree/tree_model.h GetNext:         */
/*   missing -> default child; else fvalue < split_cond -> left]                               */
/* margins_out: n x K initialised by caller to the base margin; leaves_out: n x n_trees or NULL */
/* ------------------------------------------------------------------------------------------ */
void orc_predict(const float* X, int64_t n, int32_t F, int32_t K, int32_t n_trees, int32_t tree_begin, int32_t tree_end,
                 const int64_t* tree_offset, const int32_t* tree_info, const int32_t* left, const int32_t* right,
                 const int32_t* split_index, const uint8_t* default_left, const float* split_cond,
                 float* margins_out, int32_t* leaves_out) {
  (void)n_trees;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < n; ++r) {
    const float* x = X + r * F;
    for (int t = tree_begin; t < tree_end; ++t) {
      int64_t base = tree_offset[t]; int nid = 0;
      while (left[base + nid] != -1) {
        int64_t gi = base + nid;
        int f = split_index[gi];
        float v = f < F ? x[f] : NAN;
        if (isnan(v)) nid = default_left[gi] ? left[gi] : right[gi];
        else nid = v < split_cond[gi] ? left[gi] : right[gi];
      }
      if (margins_out) margins_out[r * K + tree_info[t]] += split_cond[base + nid];
      if (leaves_out) leaves_out[r * (int64_t)(tree_end - tree_begin) + (t - tree_begin)] = nid;
    }
  }
}

void orc_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}
int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}


/* ------------------------------------------------------------------------------------------ */
/* Prediction contributions, brute force.  [UPSTREAM src/predictor/cpu_treeshap.cc computes the same quantity with the      */
/* polynomial-time Tree SHAP recursion]  Definition: the value of a feature subset S for one tree is the expectation of the */
/* tree's output when only the features in S are known -- at a split on a known feature follow the row, otherwise average  */
/* both children weighted by their cover (sum_hess).  phi_j is the Shapley value of feature j for that game, phi[F] = v({}) */
/* (+ base margin).  Enumerates all 2^F subsets: test sizes only (F <= 12).  Independent of the recursion it checks.       */
/* ------------------------------------------------------------------------------------------ */
static double shap_expect(const int32_t* left, const int32_t* right, const int32_t* split_index, const uint8_t* default_left,
                          const float* split_cond, const float* sum_hess, int64_t base, int node, const float* x, unsigned known) {
  const int64_t i = base + node;
  if (left[i] < 0) return (double)split_cond[i];
  const int f = split_index[i];
  if (known & (1u << f)) {
    const float v = x[f];
    const int go_left = (v != v) ? default_left[i] != 0 : v < split_cond[i];
    return shap_expect(left, right, split_index, default_left, split_cond, sum_hess, base, go_left ? left[i] : right[i], x, known);
  }
  const double hl = sum_hess[base + left[i]], hr = sum_hess[base + right[i]];
  return (hl * shap_expect(left, right, split_index, default_left, split_cond, sum_hess, base, left[i], x, known) +
          hr * shap_expect(left, right, split_index, default_left, split_cond, sum_hess, base, right[i], x, known)) / (double)sum_hess[i];
}

void orc_shap_bruteforce(const float* X, int64_t n, int32_t F, int32_t K, int32_t tree_begin, int32_t tree_end, const int64_t* tree_offset,
                         const int32_t* tree_info, const int32_t* left, const int32_t* right, const int32_t* split_index,
                         const uint8_t* default_left, const float* split_cond, const float* sum_hess, float base_margin, double* out) {
  const unsigned nsub = 1u << F;
  double* fact = (double*)malloc(sizeof(double) * (F + 1));
  fact[0] = 1.0; for (int i = 1; i <= F; ++i) fact[i] = fact[i - 1] * i;
#pragma omp parallel for schedule(dynamic, 4)
  for (int64_t r = 0; r < n; ++r) {
    double* v = (double*)malloc(sizeof(double) * nsub);
    const float* x = X + r * F;
    double* phi_row = out + r * K * (F + 1);
    for (int k = 0; k < K; ++k) { for (int j = 0; j <= F; ++j) phi_row[k * (F + 1) + j] = 0.0; phi_row[k * (F + 1) + F] = base_margin; }
    for (int t = tree_begin; t < tree_end; ++t) {
      double* phi = phi_row + tree_info[t] * (F + 1);
      for (unsigned S = 0; S < nsub; ++S) v[S] = shap_expect(left, right, split_index, default_left, split_cond, sum_hess, tree_offset[t], 0, x, S);
      phi[F] += v[0];
      for (int j = 0; j < F; ++j)
        for (unsigned S = 0; S < nsub; ++S) {
          if (S & (1u << j)) continue;
          const int s = __builtin_popcount(S);
          phi[j] += fact[s] * fact[F - s - 1] / fact[F] * (v[S | (1u << j)] - v[S]);
        }
    }
    free(v);
  }
  free(fact);
}
