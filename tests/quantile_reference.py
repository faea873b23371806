"""Host restatement of reg:quantileerror (parameters, gradients, the per-target leaf refresh, the base score, the quantile
metric) -- TEST INFRASTRUCTURE.  It generalises tests/absoluteerror_reference.py, whose select rules it reuses.

Upstream semantics [UPSTREAM-RECALL: src/objective/quantile_obj.cu QuantileRegression, src/metric/elementwise_metric.cu
QuantileError, src/common/quantile_loss_utils.h QuantileLossParam]:
- quantile_alpha holds Q >= 1 values, each in [0, 1]; the model has Q outputs per row from one label column, one tree per output
  per round (`tree_info` = the output), `num_target = Q` and `num_class = 0` in its documents, and predicts (n, Q);
- target j of row i: d = fl(m[i][j] - y[i]); g = fl(fl(1 - alpha_j) w) when d >= 0, else fl(-alpha_j w); h = w;
- after each tree of output j is grown, every leaf holding rows with h != 0 takes fl(q * lr), q the alpha_j-quantile of the
  residuals fl(y - m[:, j]) of those rows (absoluteerror_reference's rules: upstream `Quantile` without weights, the h_q rule with);
- the base score, when not given: mean_j q_j, q_j the (weighted) alpha_j-quantile of the labels, times sw / (sw + 1e-6) with sw
  the weight sum (the row count without weights), in double, rounded to float once [UPSTREAM-RECALL: QuantileRegression::
  InitEstimation averages the per-alpha quantiles into one scalar];
- the quantile metric: sum_i sum_j fl(w_i * pinball_j(fl(y_i - p_ij))) / (Q sum_i w_i), pinball_j(d) = fl(alpha_j d) for d >= 0,
  else fl(fl(alpha_j - 1) d), the sums in double.

The product's deviations, restated here: each target's trees grow on the fixed-point grid of that target's own gradients
(without a per-tree or gradient-based row sample), and on N GPUs the quantiles are taken over every rank's rows.

`QuantileTrainer` grows each output's trees with the oracle's unchanged squared-error trainer on carrier labels
c = (d >= 0 ? fl(alpha - 1) : alpha) with weights h: at margin 0 squared error gives (fl(-c h), h), exactly the quantile pairs.
"""
import re

import numpy as np

import absoluteerror_reference as A
from split_reference import grad_bits_for, scales_for

f32 = np.float32


class QuantileAlphaError(ValueError):
    pass


def parse_alpha(v):
    """quantile_alpha as the engine reads it: a number, "(0.1,0.5,0.9)", "[0.1, 0.5, 0.9]", a list, tuple or numpy array."""
    if isinstance(v, np.ndarray):
        v = v.tolist() if v.ndim else v.item()
    if isinstance(v, (list, tuple)):
        v = "(" + ",".join(str(x) for x in v) + ")"
    out = []
    for tok in re.split(r"[,()\[\]\s]+", str(v)):
        if not tok:
            continue
        try:
            a = f32(float(tok))
        except ValueError:
            raise QuantileAlphaError("Invalid value for parameter quantile_alpha: %s" % v)
        if not (0.0 <= a <= 1.0):
            raise QuantileAlphaError("quantile_alpha must be in [0, 1] (got %s)" % tok)
        out.append(a)
    if not out:
        raise QuantileAlphaError("quantile_alpha must not be empty")
    return np.array(out, np.float32)


def gradient(margin, y, alpha, weight=None, keep=None):
    """float32 (n, Q, 2): the quantile pairs of every target at margins (n, Q), (0, 0) outside the row sample."""
    alpha = np.asarray(alpha, np.float32)
    m = np.asarray(margin, np.float32).reshape(len(y), len(alpha))
    y = np.asarray(y, np.float32)
    w = np.ones(len(y), np.float32) if weight is None else np.asarray(weight, np.float32)
    d = (m - y[:, None]).astype(np.float32)
    g = np.where(d >= 0, (f32(1) - alpha)[None, :] * w[:, None], (-alpha)[None, :] * w[:, None]).astype(np.float32)
    h = np.repeat(w[:, None], len(alpha), axis=1)
    if keep is not None:
        g[~keep] = 0
        h[~keep] = 0
    return np.stack([g, h], axis=2).astype(np.float32)


def carriers(margin_j, y, alpha_j):
    """Squared-error labels whose gradient at margin 0 is the target's quantile g (per unit weight)."""
    d = (np.asarray(margin_j, np.float32) - np.asarray(y, np.float32)).astype(np.float32)
    return np.where(d >= 0, f32(f32(alpha_j) - f32(1)), f32(alpha_j)).astype(np.float32)


def base_score(y, alpha, weight=None):
    qs = [A.segmented_quantile(y, None, weight, 1, float(a))[0] for a in np.asarray(alpha, np.float32)]
    meanq = 0.0
    for q in qs:                              # in order, in double, as the engine sums them
        meanq += 0.0 if np.isnan(q) else float(q)
    meanq /= len(qs)
    sw = float(len(y)) if weight is None else float(np.cumsum(np.asarray(weight, np.float64))[-1])     # sequential
    return f32(meanq * sw / (sw + 1e-6))


def pinball(y, pred, alpha, weight=None):
    """The quantile metric of predictions (n, Q)."""
    alpha = np.asarray(alpha, np.float32)
    y = np.asarray(y, np.float32)
    p = np.asarray(pred, np.float32).reshape(len(y), len(alpha))
    w = np.ones(len(y), np.float32) if weight is None else np.asarray(weight, np.float32)
    d = (y[:, None] - p).astype(np.float32)
    loss = np.where(d >= 0, alpha[None, :] * d, (alpha - f32(1))[None, :] * d).astype(np.float32)
    num = np.sum((loss * w[:, None]).astype(np.float32), dtype=np.float64)
    return num / (len(alpha) * np.sum(w, dtype=np.float64))


def refresh(leaf_of_row, resid, h, weighted, sh, alpha):
    """{leaf nid: q} over the rows with h != 0, at the target's alpha."""
    return A.refresh(leaf_of_row, resid, h, weighted, sh, float(f32(alpha)))


class QuantileTrainer:
    """One boosting round per update(), as csrc/booster.cu update_one_iter runs it for this objective with one tree per output
    per round (num_parallel_tree = 1, booster=gbtree): the round's pairs of every target at the margins before the round, then
    per target j its tree grown by its own oracle trainer from the carriers, its leaves refreshed to fl(q * eta) at alpha_j from
    fl(y - m[:, j]), and column j advanced in float32.  Uniform row sampling draws one sample per round, shared by the targets."""

    def __init__(self, params, X, y, weight=None, base_margin=None, cuts=None, bins=None):
        from oracle import gbt_oracle as O
        from forest_reference import row_mask
        self.O, self.row_mask = O, row_mask
        self.params = dict(params)
        assert int(params.get("num_parallel_tree", 1)) == 1 and params.get("booster", "gbtree") == "gbtree"
        self.alpha = parse_alpha(params["quantile_alpha"])
        self.Q = len(self.alpha)
        self.X = np.ascontiguousarray(X, np.float32)
        self.y = np.asarray(y, np.float32)
        self.weight = None if weight is None else np.asarray(weight, np.float32)
        n = len(self.y)
        self.lr = f32(float(params.get("eta", 0.3)))
        drop = ("objective", "subsample", "eval_metric", "base_score", "quantile_alpha")
        op = {k: v for k, v in params.items() if k not in drop}
        op.update(objective="reg:squarederror", base_score=0.5, eta=float(self.lr))
        self.t = []
        for _ in range(self.Q):
            t = O.Trainer(op, X=self.X, y=np.zeros(n, np.float32), weights=np.ones(n, np.float32), cuts=cuts, bins=bins, base_score=0.5)
            t.set_device_grid()
            self.t.append(t)
        self.base_score = f32(params["base_score"]) if "base_score" in params else base_score(self.y, self.alpha, self.weight)
        self.m = (np.full((n, self.Q), self.base_score, np.float32) if base_margin is None
                  else np.asarray(base_margin, np.float32).reshape(n, self.Q).copy())
        self.trees = []                           # model order: (target, that target's oracle tree id)
        self.leaves = {}                          # model tree -> {nid: refreshed value}
        self.rounds = 0

    def update(self):
        n = len(self.y)
        keep = self.row_mask(int(self.params.get("seed", 0)), self.rounds, 0, n, float(self.params.get("subsample", 1.0)))
        m0 = self.m.copy()
        gp = gradient(m0, self.y, self.alpha, self.weight, keep)
        for j in range(self.Q):
            t = self.t[j]
            resid = (self.y - m0[:, j]).astype(np.float32)
            t.y[:] = carriers(m0[:, j], self.y, self.alpha[j])
            t.w[:] = gp[:, j, 1]
            t.set_margins(np.zeros(n, np.float32))
            t.update()
            model = t.model()
            tid = model.num_trees - 1
            leaf = self.O.predict_leaf(model, self.X, tid, tid + 1)[:, 0]
            h = gp[:, j, 1]
            sh = scales_for(np.max(np.abs(gp[:, j, 0])), np.max(h), grad_bits_for(n))[1]
            q = refresh(leaf, resid, h, self.weight is not None, sh, self.alpha[j])
            vals = {nid: f32(v * self.lr) for nid, v in q.items()}
            value = model.tree(tid)["split_cond"].copy()
            for nid, v in vals.items():
                value[nid] = v
            self.leaves[len(self.trees)] = vals
            self.trees.append((j, tid))
            self.m[:, j] = (self.m[:, j] + value[leaf]).astype(np.float32)
        self.rounds += 1

    def model(self):
        """The model in the layout booster_export_model returns: trees in model order, tree_info = output."""
        sub = [t.model() for t in self.t]
        out = self.O.Model()
        keys_i = ("left", "right", "parent", "split_index", "split_bin")
        keys_f = ("split_cond", "base_weight", "loss_chg", "sum_hess")
        parts = {k: [] for k in keys_i + keys_f + ("default_left",)}
        offs = [0]
        for t, (j, tid) in enumerate(self.trees):
            m = sub[j]
            a, b = int(m["tree_offset"][tid]), int(m["tree_offset"][tid + 1])
            for k in parts:
                parts[k].append(np.asarray(m[k][a:b]).copy())
            for nid, v in self.leaves[t].items():
                parts["split_cond"][-1][nid] = v
            offs.append(offs[-1] + b - a)
        for k in parts:
            dt = np.float32 if k in keys_f else (np.uint8 if k == "default_left" else np.int32)
            out[k] = np.concatenate(parts[k]).astype(dt) if parts[k] else np.zeros(0, dt)
        out["tree_offset"] = np.array(offs, np.int64)
        out["tree_info"] = np.array([j for j, _ in self.trees], np.int32)
        out["base_score"] = float(self.base_score)
        out["num_class"] = self.Q
        return out

    def margins(self):
        return self.m
