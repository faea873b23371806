"""Host restatement of reg:absoluteerror (gradients, the per-leaf quantile refresh, the base score) -- TEST INFRASTRUCTURE.

Upstream semantics [UPSTREAM-RECALL: src/objective/regression_obj.cu MeanAbsoluteError, src/objective/adaptive.{h,cc,cu},
src/common/stats.h Quantile / WeightedQuantile]: g = sign(m - y) w, h = w; after each tree is grown, every leaf holding rows
with h != 0 takes fl(q * lr), q the 0.5-quantile of the float residuals fl(y - m) of those rows.

The product's rule, restated here:
- unweighted: upstream's `Quantile` in its own types (float order statistics, double interpolation weight, float difference);
- weighted: the first sorted residual whose cumulative h_q reaches alpha * total, h_q = rint(h * sh) on the fixed-point grid of
  the round's histograms (`split_reference.scales_for`), so every cumulative weight is an exact integer.  Upstream accumulates a
  float CDF instead (`upstream_weighted_quantile`); the two agree unless that CDF lands within rounding of alpha * total;
- -0.0 residuals count as +0.0, every NaN as one value above +inf, and the values are ordered by their order-preserving
  uint32 keys.

`AbsErrorTrainer` grows the trees with the oracle's unchanged trainer, fed squared-error carrier labels -sign(m - y) and weights
h, whose gradient pairs at margin 0 equal the absolute-error pairs exactly, then refreshes the leaves here and advances the
margins in float32.
"""
import numpy as np

from split_reference import grad_bits_for, scales_for

f32 = np.float32


def keys(v):
    """Order-preserving uint32 keys of float32 values, -0.0 taken as +0.0 and every NaN as the positive quiet NaN."""
    v = np.asarray(v, np.float32)
    b = np.ascontiguousarray(v).view(np.uint32).copy()
    b[b == np.uint32(0x80000000)] = 0
    b[np.isnan(v)] = 0x7FC00000               # every NaN: one value above +inf
    neg = (b & np.uint32(0x80000000)) != 0
    return np.where(neg, ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def _sorted(v):
    v = np.asarray(v, np.float32)
    k = keys(v)
    order = np.argsort(k, kind="stable")
    out = v[order].copy()
    out[out == 0] = f32(0.0)                  # -0.0 -> +0.0
    return out, order


def quantile(v, alpha=0.5):
    """Upstream common::Quantile on float values: the ends clamp, else v0 + d (v1 - v0) with d in double, v1 - v0 in float."""
    s, _ = _sorted(v)
    n = float(len(s))
    if n == 0:
        return f32(np.nan)
    if alpha <= 1.0 / (n + 1.0):
        return s[0]
    if alpha >= n / (n + 1.0):
        return s[-1]
    x = alpha * (n + 1.0)
    k = np.floor(x) - 1.0
    d = (x - 1.0) - k
    v0, v1 = s[int(k)], s[int(k) + 1]
    with np.errstate(over="ignore", invalid="ignore"):
        diff = f32(v1 - v0)
        return f32(float(v0) + d * float(diff))


def weighted_quantile_hq(v, hq, alpha=0.5):
    """The product's weighted rule on integer weights hq: the first sorted value whose cumulative hq reaches
    ceil(alpha * total); the smallest value when the total (or that target) is 0."""
    s, order = _sorted(v)
    if len(s) == 0:
        return f32(np.nan)
    cum = np.cumsum(np.asarray(hq, np.int64)[order])
    total = int(cum[-1])
    c = int(np.ceil(alpha * float(total)))
    if total == 0 or c < 1:
        return s[0]
    return s[int(np.searchsorted(cum, c, side="left"))]


def upstream_weighted_quantile(v, w, alpha=0.5):
    """Upstream common::WeightedQuantile: a float CDF accumulated in sorted order, thresh = float(cdf[-1] * alpha), the first
    position with cdf >= thresh, clamped to n - 1."""
    s, order = _sorted(v)
    n = len(s)
    if n == 0:
        return f32(np.nan)
    cdf = np.cumsum(np.asarray(w, np.float32)[order], dtype=np.float32)     # add.accumulate: sequential, in float
    thresh = f32(float(cdf[-1]) * alpha)
    idx = int(np.searchsorted(cdf, thresh, side="left"))
    return s[min(idx, n - 1)]


def h_q(h, sh):
    """The histograms' fixed-point hessian: rint(h * sh) (round half to even), sh a power of two."""
    return np.rint(np.asarray(h, np.float32) * f32(sh)).astype(np.int64)


def weight_scale(w, n):
    """sh of a matrix of n rows whose largest hessian is max(w) (csrc/tree.cu scales_kernel)."""
    mw = f32(np.max(w)) if len(w) else f32(0)
    return scales_for(0.0, mw, grad_bits_for(n))[1]


def segmented_quantile(values, segments=None, weights=None, n_segments=1, alpha=0.5):
    """What XGB200SegmentedQuantile returns: per segment, NaN when it has no rows; rows with segment -1 or weight 0 left out."""
    v = np.asarray(values, np.float32)
    n = len(v)
    seg = np.zeros(n, np.int64) if segments is None else np.asarray(segments, np.int64)
    w = None if weights is None else np.asarray(weights, np.float32)
    keep = seg >= 0
    if w is not None:
        keep &= w != 0
        hq = h_q(w, weight_scale(w, n))
    out = np.full(n_segments, np.nan, np.float32)
    order = np.argsort(seg, kind="stable")
    bounds = np.searchsorted(seg[order], np.arange(n_segments + 1))
    for s in range(n_segments):
        rows = order[bounds[s]:bounds[s + 1]]
        rows = rows[keep[rows]]
        if len(rows) == 0:
            continue
        out[s] = quantile(v[rows], alpha) if w is None else weighted_quantile_hq(v[rows], hq[rows], alpha)
    return out


def gradient(margin, y, weight=None, keep=None):
    """float32 (n, 2): (sign(m - y) w, w), (0, 0) outside the row sample."""
    m = np.asarray(margin, np.float32)
    y = np.asarray(y, np.float32)
    w = np.ones(len(y), np.float32) if weight is None else np.asarray(weight, np.float32)
    g = np.sign(m - y).astype(np.float32) * w
    h = w.copy()
    if keep is not None:
        g[~keep] = 0
        h[~keep] = 0
    return np.stack([g, h], axis=1).astype(np.float32)


def base_score(y, weight=None):
    """The estimated base score: the median of the labels (weighted on the weights' fixed-point grid)."""
    q = segmented_quantile(y, None, weight, 1, 0.5)[0]
    return f32(0.0) if np.isnan(q) else q


def refresh(leaf_of_row, resid, h, weighted, sh, alpha=0.5):
    """{leaf nid: q} over the rows with h != 0."""
    use = np.asarray(h) != 0
    out = {}
    for nid in np.unique(leaf_of_row[use]):
        rows = np.nonzero(use & (leaf_of_row == nid))[0]
        out[int(nid)] = weighted_quantile_hq(resid[rows], h_q(h[rows], sh), alpha) if weighted else quantile(resid[rows], alpha)
    return out


class AbsErrorTrainer:
    """One boosting round per update(), as csrc/booster.cu update_one_iter runs it for this objective:
      * booster=dart: the drop set, the dropped trees' new weights and the gradient margin without them, in the float steps of
        tests/dart_reference.py; the new tree's leaves enter the margin times the round's new-tree weight;
      * num_parallel_tree = P: P trees on the round's gradients, tree j on its own row sample (tests/forest_reference.py
        row_mask: tree 0 the single-tree stream), with leaves fl(eta / P) * w and the refresh's lr = fl(eta / P);
      * every tree: the absolute-error pairs of its sample at the round's gradient margin, grown by the oracle from their
        carriers, its leaves refreshed to fl(q * lr) from the residuals fl(y - m) at that margin, the margins advanced in float32.
    The oracle numbers its trees in growth order, which is the model order at one class."""

    def __init__(self, params, X, y, weight=None, base_margin=None, cuts=None, bins=None):
        from oracle import gbt_oracle as O
        from dart_reference import dart_param
        from forest_reference import forest_eta
        self.O = O
        self.params = dict(params)
        self.X = np.ascontiguousarray(X, np.float32)
        self.y = np.asarray(y, np.float32)
        self.weight = None if weight is None else np.asarray(weight, np.float32)
        n = len(self.y)
        self.P = int(params.get("num_parallel_tree", 1))
        self.eta = float(params.get("eta", 0.3))
        self.lr = forest_eta(self.eta, self.P)
        self.dart = dart_param(params) if params.get("booster") == "dart" else None
        drop = ("objective", "subsample", "eval_metric", "base_score", "num_parallel_tree", "booster", "rate_drop", "skip_drop", "one_drop",
                "sample_type", "normalize_type")
        op = {k: v for k, v in params.items() if k not in drop}
        op.update(objective="reg:squarederror", base_score=0.5, eta=float(self.lr))
        self.t = O.Trainer(op, X=self.X, y=np.zeros(n, np.float32), weights=np.ones(n, np.float32), cuts=cuts, bins=bins, base_score=0.5)
        self.t.set_device_grid()
        self.base_score = f32(params["base_score"]) if "base_score" in params else base_score(self.y, self.weight)
        self.m = np.full(n, self.base_score, np.float32) if base_margin is None else np.asarray(base_margin, np.float32).copy()
        self.leaves = {}                          # tree -> {nid: refreshed value}
        self.rows, self.values = [], []           # per tree: every row's leaf, the tree's node values after the refresh
        self.weights = []                         # per tree: its weight in the margin (booster=dart; else 1)
        self.rounds = 0

    def _tree_values(self, t):
        return self.values[t][self.rows[t]]

    def _grow(self, gp, resid):
        """One tree on the pairs gp; returns every row's refreshed leaf value."""
        n = len(self.y)
        self.t.y[:] = -np.sign(gp[:, 0]).astype(np.float32)
        self.t.w[:] = gp[:, 1]
        self.t.set_margins(np.zeros(n, np.float32))
        self.t.update()
        model = self.t.model()
        tid = model.num_trees - 1
        leaf = self.O.predict_leaf(model, self.X, tid, tid + 1)[:, 0]
        h = gp[:, 1]
        sh = scales_for(np.max(np.abs(gp[:, 0])), np.max(h), grad_bits_for(n))[1]
        q = refresh(leaf, resid, h, self.weight is not None, sh)
        vals = {nid: f32(v * self.lr) for nid, v in q.items()}
        self.leaves[tid] = vals
        value = model.tree(tid)["split_cond"].copy()
        for nid, v in vals.items():
            value[nid] = v
        self.rows.append(leaf)
        self.values.append(value)
        return value[leaf]

    def update(self):
        from dart_reference import drop_set, normalisation
        from forest_reference import row_mask
        n = len(self.y)
        seed, rnd = int(self.params.get("seed", 0)), self.rounds
        w_new = f32(1)
        m_grad = self.m
        if self.dart is not None:
            D = drop_set(self.weights, rnd, seed, self.dart)
            factor, w_new = normalisation(len(D), self.eta, 1, self.dart["normalize_type"])
            m_grad = self.m.copy()
            for j in D:                          # ascending: m_drop -= fl(w * leaf), m_full += fl(c * leaf), c = fl(w' - w)
                v = self._tree_values(j)
                w = f32(self.weights[j])
                w2 = f32(w * factor)
                m_grad = m_grad - w * v
                self.m = self.m + f32(w2 - w) * v
                self.weights[j] = w2
        m_grad = np.asarray(m_grad, np.float32).copy()
        resid = (self.y - m_grad).astype(np.float32)
        full = gradient(m_grad, self.y, self.weight)
        for j in range(self.P):
            gp = full.copy()
            keep = row_mask(seed, rnd, j, n, float(self.params.get("subsample", 1.0)))
            gp[~keep] = 0
            v = self._grow(gp, resid)
            self.m = (self.m + (v if self.dart is None else w_new * v)).astype(np.float32)
            self.weights.append(w_new)
        self.rounds += 1

    def model(self):
        m = self.t.model()
        for tid, vals in self.leaves.items():
            off = int(m["tree_offset"][tid])
            for nid, v in vals.items():
                m["split_cond"][off + nid] = v
        m["base_score"] = float(self.base_score)
        return m

    def margins(self):
        return self.m.reshape(-1, 1)
