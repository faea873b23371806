"""ctypes wrapper around oracle/libgbt_oracle.so -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The oracle is the CPU restatement of the reference's `tree_method=hist` path (see the header of
gbt_oracle.c for the reference/upstream files each function follows).  Only tests/,
`__graft_entry__.smoke()` and bench.py's cpu_baseline / `--impl reference` leg may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgbt_oracle.so")
_SRC = os.path.join(_HERE, "gbt_oracle.c")

OBJECTIVES = {
    "reg:squarederror": 0, "reg:linear": 0, "binary:logistic": 1, "reg:logistic": 2,
    "binary:logitraw": 3, "multi:softprob": 4, "multi:softmax": 5,
    "reg:squaredlogerror": 6, "reg:pseudohubererror": 7, "count:poisson": 8, "reg:gamma": 9, "reg:tweedie": 10, "binary:hinge": 11,
}


def build(force=False):
    """Compile the oracle with gcc (recipe committed here; output is git-ignored)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        # -ffp-contract=off: the split gains round every product before the add, as upstream's CPU code (and the product) do;
        # a compiler that fuses them (gcc on aarch64 does by default) would move loss_chg by an ulp
        subprocess.check_call(["gcc", "-O3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", "-o", _SO, _SRC, "-lm"])
    return _SO


class OrcSplit(C.Structure):
    _fields_ = [("loss_chg", C.c_float), ("findex", C.c_int32), ("split_value", C.c_float), ("split_bin", C.c_int32),
                ("default_left", C.c_int32), ("GL", C.c_double), ("HL", C.c_double), ("GR", C.c_double), ("HR", C.c_double)]


class OrcParams(C.Structure):
    _fields_ = [
        ("objective", C.c_int32), ("num_class", C.c_int32), ("max_depth", C.c_int32),
        ("max_leaves", C.c_int32), ("max_bin", C.c_int32), ("grow_policy", C.c_int32),
        ("nthread", C.c_int32), ("seed", C.c_uint32),
        ("eta", C.c_float), ("lambda_", C.c_float), ("alpha", C.c_float), ("gamma", C.c_float),
        ("min_child_weight", C.c_float), ("max_delta_step", C.c_float), ("scale_pos_weight", C.c_float),
        ("subsample", C.c_float), ("colsample_bytree", C.c_float), ("colsample_bylevel", C.c_float),
        ("colsample_bynode", C.c_float),
        ("huber_slope", C.c_float), ("tweedie_variance_power", C.c_float), ("poisson_max_delta_step", C.c_float),
    ]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.orc_trainer_create.restype = C.c_void_p
        L.orc_trainer_create.argtypes = [C.POINTER(OrcParams), C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_int32]
        L.orc_trainer_free.argtypes = [C.c_void_p]
        L.orc_update_one_iter.argtypes = [C.c_void_p]
        L.orc_num_trees.argtypes = [C.c_void_p]
        L.orc_num_nodes.argtypes = [C.c_void_p]
        L.orc_num_nodes.restype = C.c_int64
        L.orc_get_base_score.argtypes = [C.c_void_p]
        L.orc_get_base_score.restype = C.c_float
        L.orc_margins.argtypes = [C.c_void_p]
        L.orc_margins.restype = C.POINTER(C.c_float)
        L.orc_gpair.argtypes = [C.c_void_p]
        L.orc_gpair.restype = C.POINTER(C.c_float)
        L.orc_export_model.argtypes = [C.c_void_p] + [C.c_void_p] * 12
        L.orc_make_cuts.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]
        L.orc_bin.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_gradient.argtypes = [C.POINTER(OrcParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.orc_base_score.argtypes = [C.POINTER(OrcParams), C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_base_score.restype = C.c_float
        for fn, nargs in (("orc_calc_weight", 2), ("orc_calc_gain", 2), ("orc_calc_split_gain", 4)):
            getattr(L, fn).argtypes = [C.POINTER(OrcParams)] + [C.c_double] * nargs
            getattr(L, fn).restype = C.c_float
        L.orc_prob_to_margin.argtypes = [C.POINTER(OrcParams), C.c_float]
        L.orc_prob_to_margin.restype = C.c_float
        L.orc_build_hist.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                     C.c_int32, C.c_void_p]
        L.orc_build_hist_fixed.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.orc_predict.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 9
        L.orc_num_threads.restype = C.c_int
        L.orc_set_quant_bits.argtypes = [C.c_void_p, C.c_int32]
        L.orc_set_monotone.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.orc_set_interaction.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.orc_set_margins.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_eval_split.argtypes = [C.POINTER(OrcParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                     C.c_double, C.c_double, C.c_float, C.POINTER(OrcSplit)]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def make_params(params):
    """Translate an xgboost-style parameter dict (aliases eta/gamma/lambda/alpha accepted) into OrcParams."""
    g = params.get
    obj = g("objective", "reg:squarederror")
    if obj not in OBJECTIVES:
        raise ValueError("oracle: unsupported objective %r" % obj)
    p = OrcParams()
    p.objective = OBJECTIVES[obj]
    p.num_class = int(g("num_class", 1)) if p.objective in (4, 5) else 1
    p.max_depth = int(g("max_depth", 6))
    p.max_leaves = int(g("max_leaves", 0))
    p.max_bin = int(g("max_bin", 256))
    p.grow_policy = 1 if g("grow_policy", "depthwise") == "lossguide" else 0
    p.nthread = int(g("nthread", 0) or 0)
    p.seed = int(g("seed", 0))
    p.eta = float(g("eta", g("learning_rate", 0.3)))
    p.lambda_ = float(g("lambda", g("reg_lambda", 1.0)))
    p.alpha = float(g("alpha", g("reg_alpha", 0.0)))
    p.gamma = float(g("gamma", g("min_split_loss", 0.0)))
    p.min_child_weight = float(g("min_child_weight", 1.0))
    p.max_delta_step = float(g("max_delta_step", 0.0))
    p.scale_pos_weight = float(g("scale_pos_weight", 1.0))
    p.subsample = float(g("subsample", 1.0))
    p.colsample_bytree = float(g("colsample_bytree", 1.0))
    p.colsample_bylevel = float(g("colsample_bylevel", 1.0))
    p.colsample_bynode = float(g("colsample_bynode", 1.0))
    p.huber_slope = float(g("huber_slope", 1.0))
    p.tweedie_variance_power = float(g("tweedie_variance_power", 1.5))
    if obj == "count:poisson":          # upstream learner.cc: max_delta_step defaults to 0.7 for count:poisson (objective AND tree)
        if g("max_delta_step") is None:
            p.max_delta_step = 0.7
        p.poisson_max_delta_step = p.max_delta_step
    else:
        p.poisson_max_delta_step = 0.7
    return p


def make_cuts(X, max_bin=256, weights=None):
    X = np.ascontiguousarray(X, dtype=np.float32)
    n, F = X.shape
    cut_ptrs = np.zeros(F + 1, np.int32)
    cut_vals = np.zeros(F * 256, np.float32)
    min_vals = np.zeros(F, np.float32)
    hm = C.c_int32(0)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    tot = lib().orc_make_cuts(_p(X), n, F, _p(w), int(max_bin), _p(cut_ptrs), _p(cut_vals), _p(min_vals), C.byref(hm))
    return cut_ptrs, cut_vals[:tot].copy(), min_vals, bool(hm.value)


def bin_matrix(X, cut_ptrs, cut_vals):
    X = np.ascontiguousarray(X, dtype=np.float32)
    n, F = X.shape
    bins = np.empty((n, F), np.uint8)
    lib().orc_bin(_p(X), n, F, _p(cut_ptrs), _p(cut_vals), _p(bins))
    return bins


def gradient(params, margins, labels, weights=None):
    p = make_params(params)
    K = max(1, p.num_class)
    margins = np.ascontiguousarray(margins, np.float32).reshape(-1, K)
    n = margins.shape[0]
    labels = np.ascontiguousarray(labels, np.float32)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    gp = np.empty((n, K, 2), np.float32)
    rc = lib().orc_gradient(C.byref(p), _p(margins), _p(labels), _p(w), n, _p(gp))
    if rc == -1:
        raise ValueError("label must be in [0,1] for logistic regression")
    if rc == -2:
        raise ValueError("SoftmaxMultiClassObj: label must be in [0, num_class).")
    return gp


def build_hist(bins, cut_ptrs, gpair, rows=None, has_missing=False):
    """Reference-faithful histogram: float gpair accumulated in double. Returns (total_bins, 2) float64."""
    bins = np.ascontiguousarray(bins, np.uint8)
    n, F = bins.shape
    gpair = np.ascontiguousarray(gpair, np.float32).reshape(n, 2)
    hist = np.zeros((int(cut_ptrs[F]), 2), np.float64)
    r = None if rows is None else np.ascontiguousarray(rows, np.uint32)
    lib().orc_build_hist(_p(bins), F, _p(np.ascontiguousarray(cut_ptrs, np.int32)), _p(gpair), 2, _p(r),
                         n if r is None else len(r), int(has_missing), _p(hist))
    return hist


def build_hist_fixed(bins, gq, hq, rows=None):
    """Fixed-point mirror: exact int64 sums of int32 quantised gradients. Returns (F, 256, 2) int64."""
    bins = np.ascontiguousarray(bins, np.uint8)
    n, F = bins.shape
    gq = np.ascontiguousarray(gq, np.int32)
    hq = np.ascontiguousarray(hq, np.int32)
    hist = np.zeros((F, 256, 2), np.int64)
    r = None if rows is None else np.ascontiguousarray(rows, np.uint32)
    lib().orc_build_hist_fixed(_p(bins), F, _p(gq), _p(hq), _p(r), n if r is None else len(r), _p(hist))
    return hist


def eval_split(params, hist, cut_ptrs, cut_vals, min_vals, G, H, root_gain, feat_mask=None):
    """Best unconstrained split of one node (EnumerateSplit over every feature): hist is (total_bins, 2) float64 (g, h), G, H
    the node totals, root_gain its float gain.  Returns the oracle's Split as a dict."""
    p = make_params(params)
    hist = np.ascontiguousarray(hist, np.float64)
    ptrs = np.ascontiguousarray(cut_ptrs, np.int32)
    vals = np.ascontiguousarray(cut_vals, np.float32)
    mins = np.ascontiguousarray(min_vals, np.float32)
    mask = None if feat_mask is None else np.ascontiguousarray(feat_mask, np.uint8)
    out = OrcSplit()
    lib().orc_eval_split(C.byref(p), _p(hist), _p(ptrs), _p(vals), _p(mins), len(ptrs) - 1, _p(mask), float(G), float(H),
                         C.c_float(root_gain), C.byref(out))
    return {k: getattr(out, k) for k, _ in OrcSplit._fields_}


class Model(dict):
    """Flat tree arrays: tree_offset, tree_info, left, right, parent, split_index, split_bin,
    default_left, split_cond, base_weight, loss_chg, sum_hess + base_score, num_class, num_feature."""

    def tree(self, t):
        a, b = int(self["tree_offset"][t]), int(self["tree_offset"][t + 1])
        return {k: self[k][a:b] for k in ("left", "right", "parent", "split_index", "split_bin", "default_left",
                                          "split_cond", "base_weight", "loss_chg", "sum_hess")}

    @property
    def num_trees(self):
        return len(self["tree_info"])


class Trainer:
    """Stateful oracle trainer: one `update()` = one boosting round on pre-binned data."""

    def __init__(self, params, X=None, y=None, weights=None, bins=None, cuts=None, base_score=None):
        self.params = dict(params)
        self.p = make_params(params)
        if bins is None:
            X = np.ascontiguousarray(X, np.float32)
            if cuts is None:
                cuts = make_cuts(X, self.p.max_bin, weights)
            self.cut_ptrs, self.cut_vals, self.min_vals, self.has_missing = cuts
            bins = bin_matrix(X, self.cut_ptrs, self.cut_vals)
        else:
            self.cut_ptrs, self.cut_vals, self.min_vals, self.has_missing = cuts
        self.cut_ptrs = np.ascontiguousarray(self.cut_ptrs, np.int32)
        self.cut_vals = np.ascontiguousarray(self.cut_vals, np.float32)
        self.min_vals = np.ascontiguousarray(self.min_vals, np.float32)
        self.bins = np.ascontiguousarray(bins, np.uint8)
        self.n, self.F = self.bins.shape
        self.y = np.ascontiguousarray(y, np.float32)
        self.w = None if weights is None else np.ascontiguousarray(weights, np.float32)
        if base_score is None and "base_score" in params and params["base_score"] is not None:
            base_score = float(params["base_score"])
        self.h = lib().orc_trainer_create(C.byref(self.p), _p(self.bins), self.n, self.F, _p(self.cut_ptrs),
                                          _p(self.cut_vals), _p(self.min_vals), _p(self.y), _p(self.w),
                                          int(self.has_missing), float(base_score or 0.0), int(base_score is not None))
        mc = params.get("monotone_constraints")
        if mc is not None:
            if isinstance(mc, str):
                mc = [int(t) for t in mc.strip("()[] ").split(",") if t.strip()]
            self._mono = np.ascontiguousarray(list(mc), np.int32)
            lib().orc_set_monotone(self.h, _p(self._mono), len(self._mono))
        ic = params.get("interaction_constraints")
        if ic:
            if isinstance(ic, str):
                import json
                ic = json.loads(ic.replace("(", "[").replace(")", "]"))
            sets = np.zeros((len(ic), self.F), np.uint8)
            for si, grp in enumerate(ic):
                sets[si, [int(f) for f in grp]] = 1
            self._ic = np.ascontiguousarray(sets)
            lib().orc_set_interaction(self.h, _p(self._ic), len(ic))

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_trainer_free(self.h)
            self.h = None

    @property
    def K(self):
        return max(1, self.p.num_class)

    def set_quant_bits(self, bits):
        """Study knob: emulate the product's fixed-point gradient grid with `bits` - 1 magnitude bits of g (0 = reference
        behaviour): g is rounded to 2^(bits - 1 - eg), h to 2^(bits - eh), as the product's scales_kernel does."""
        lib().orc_set_quant_bits(self.h, int(bits))

    def set_device_grid(self, n=None):
        """The grid the product trains `n` rows (default: this trainer's) on: 21 magnitude bits up to 2^20 rows, 18 above
        (csrc/engine.h grad_bits_for)."""
        n = self.n if n is None else int(n)
        self.set_quant_bits((21 if n <= (1 << 20) else 18) + 1)

    def set_margins(self, m):
        m = np.ascontiguousarray(m, np.float32).reshape(self.n, self.K)
        lib().orc_set_margins(self.h, _p(m))

    def update(self):
        rc = lib().orc_update_one_iter(self.h)
        if rc == -1:
            raise ValueError("label must be in [0,1] for logistic regression")
        if rc == -2:
            raise ValueError("SoftmaxMultiClassObj: label must be in [0, num_class).")

    def margins(self):
        ptr = lib().orc_margins(self.h)
        return np.ctypeslib.as_array(ptr, shape=(self.n, self.K)).copy()

    def gpair(self):
        ptr = lib().orc_gpair(self.h)
        return np.ctypeslib.as_array(ptr, shape=(self.n, self.K, 2)).copy()

    @property
    def base_score(self):
        return float(lib().orc_get_base_score(self.h))

    def model(self):
        nt = lib().orc_num_trees(self.h)
        nn = lib().orc_num_nodes(self.h)
        m = Model()
        m["tree_offset"] = np.zeros(nt + 1, np.int64)
        m["tree_info"] = np.zeros(nt, np.int32)
        for k in ("left", "right", "parent", "split_index", "split_bin"):
            m[k] = np.zeros(nn, np.int32)
        m["default_left"] = np.zeros(nn, np.uint8)
        for k in ("split_cond", "base_weight", "loss_chg", "sum_hess"):
            m[k] = np.zeros(nn, np.float32)
        lib().orc_export_model(self.h, _p(m["tree_offset"]), _p(m["tree_info"]), _p(m["left"]), _p(m["right"]),
                               _p(m["parent"]), _p(m["split_index"]), _p(m["split_bin"]), _p(m["default_left"]),
                               _p(m["split_cond"]), _p(m["base_weight"]), _p(m["loss_chg"]), _p(m["sum_hess"]))
        m["base_score"] = self.base_score
        m["num_class"] = self.K
        m["num_feature"] = self.F
        m["objective"] = self.params.get("objective", "reg:squarederror")
        return m


def train(params, X, y, num_boost_round, weights=None, cuts=None, bins=None):
    t = Trainer(params, X=X, y=y, weights=weights, cuts=cuts, bins=bins)
    for _ in range(num_boost_round):
        t.update()
    return t


def base_margin_of(model):
    p = make_params({"objective": model.get("objective", "reg:squarederror"), "num_class": model.get("num_class", 1)})
    return float(lib().orc_prob_to_margin(C.byref(p), float(model["base_score"])))


def predict_margin(model, X, tree_begin=0, tree_end=None, base_margin=None):
    """fp32 margins (n, K): the leaf values of trees [tree_begin, tree_end) added in tree order to the base margin, a scalar
    (default: the model's) or per row, (n,) or (n, K) like DMatrix base_margin."""
    X = np.ascontiguousarray(X, np.float32)
    n, F = X.shape
    K = int(model.get("num_class", 1))
    nt = model.num_trees if isinstance(model, Model) else len(model["tree_info"])
    tree_end = nt if tree_end is None else tree_end
    bm = base_margin_of(model) if base_margin is None else base_margin
    if np.ndim(bm) == 0:
        out = np.full((n, K), bm, np.float32)
    else:
        out = np.array(bm, np.float32).reshape(n, K)
    lib().orc_predict(_p(X), n, F, K, nt, tree_begin, tree_end, _p(model["tree_offset"]), _p(model["tree_info"]),
                      _p(model["left"]), _p(model["right"]), _p(model["split_index"]), _p(model["default_left"]),
                      _p(model["split_cond"]), _p(out), None)
    return out


def predict_leaf(model, X, tree_begin=0, tree_end=None):
    X = np.ascontiguousarray(X, np.float32)
    n, F = X.shape
    K = int(model.get("num_class", 1))
    nt = len(model["tree_info"])
    tree_end = nt if tree_end is None else tree_end
    out = np.zeros((n, tree_end - tree_begin), np.int32)
    lib().orc_predict(_p(X), n, F, K, nt, tree_begin, tree_end, _p(model["tree_offset"]), _p(model["tree_info"]),
                      _p(model["left"]), _p(model["right"]), _p(model["split_index"]), _p(model["default_left"]),
                      _p(model["split_cond"]), None, _p(out))
    return out


def shap_bruteforce(model, X, tree_begin=0, tree_end=None):
    """Exact Shapley values of the cover-weighted conditional-expectation game, by subset enumeration (F <= 12): the quantity
    Tree SHAP / Booster.predict(pred_contribs=True) computes.  Returns float64 (n, K, F + 1); last column = bias."""
    X = np.ascontiguousarray(X, np.float32)
    n, F = X.shape
    assert F <= 12, "brute force enumerates 2^F subsets"
    K = int(model.get("num_class", 1))
    nt = len(model["tree_info"])
    tree_end = nt if tree_end is None else tree_end
    out = np.zeros((n, K, F + 1), np.float64)
    L = lib()
    L.orc_shap_bruteforce.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 8 + [C.c_float, C.c_void_p]
    L.orc_shap_bruteforce(_p(X), n, F, K, tree_begin, tree_end, _p(model["tree_offset"]), _p(model["tree_info"]), _p(model["left"]),
                          _p(model["right"]), _p(model["split_index"]), _p(model["default_left"]), _p(model["split_cond"]),
                          _p(model["sum_hess"]), C.c_float(base_margin_of(model)), _p(out))
    return out


def transform(model, margins):
    """PredTransform of the objective (identity / sigmoid / softmax)."""
    obj = model.get("objective", "reg:squarederror")
    m = np.asarray(margins, np.float32)
    if obj in ("binary:logistic", "reg:logistic"):
        return (1.0 / (1.0 + np.exp(-m, dtype=np.float32))).astype(np.float32)
    if obj in ("count:poisson", "reg:gamma", "reg:tweedie"):
        return np.exp(m, dtype=np.float32)
    if obj == "binary:hinge":
        return (m > 0).astype(np.float32)
    if obj == "multi:softprob":
        e = np.exp(m - m.max(axis=1, keepdims=True), dtype=np.float32)
        return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)
    if obj == "multi:softmax":
        return m.argmax(axis=1).astype(np.float32)
    return m


def num_threads():
    return int(lib().orc_num_threads())


def set_num_threads(n):
    """Explicit OpenMP thread count for every oracle entry point (bench.py sets it: torchrun exports OMP_NUM_THREADS=1)."""
    lib().orc_set_num_threads(int(n))
    return num_threads()
