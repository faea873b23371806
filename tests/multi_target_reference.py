"""Multi-target regression restated in numpy (DESIGN.md "Multi-target regression"): a label Y of shape (n, T), one tree per
target per round, `tree_info` the target, predictions of shape (n, T).

- `gradient`: the float32 pairs of every element, (n, T, 2), and `target_absmax` each target's max|g| and max h, the
  fixed-point grid its trees grow on.  Each element is the single-target objective's pair of (y_ij, m_ij) with the row's weight
  w_i (times scale_pos_weight when y_ij == 1 under the RegLossObj family).  reg:squarederror and reg:absoluteerror use only
  IEEE-rounded float32 operations and restate the kernel bit for bit.  The logistic family and reg:squaredlogerror call expf /
  log1pf, which CUDA and numpy round differently in the last place, and the CUDA build contracts multiplies and adds of the
  pseudo-Huber pair into fused multiply-adds in a way not restated here: for these this restatement agrees to a few ulp, and
  the device test pins each target to the single-target kernel on its column instead.
- `intercept`: the estimated base_score.  Each target's Newton stump at margin 0 (sums in double), their mean in double in
  target order, then the objective's transform once; reg:absoluteerror takes the mean of the columns' weighted medians.
- `metric`: the element-wise metrics over the n x T elements, sum_i sum_j w_i l(y_ij, p_ij) / (T sum_i w_i) in double, then the
  metric's finalisation (sqrt for rmse and rmsle).
- `shapes`: what predict() returns for each kind of call.
"""
import numpy as np

import absoluteerror_reference as AR

f32 = np.float32
OBJECTIVES = ("reg:squarederror", "reg:squaredlogerror", "reg:pseudohubererror", "reg:logistic", "binary:logistic", "binary:logitraw",
              "reg:absoluteerror")
EXACT = ("reg:squarederror", "reg:absoluteerror")      # bit-exact restatements (see the module doc)
LOGISTIC = ("reg:logistic", "binary:logistic", "binary:logitraw")
METRICS = ("rmse", "rmsle", "mae", "mape", "mphe", "logloss", "error")


def sigmoid(x):
    """transform.h sigmoidf_xgb: 1 / (exp(min(-x, 88.7)) + 1 + 1e-16), in float32 (exp rounded from double)."""
    x = np.minimum(-np.asarray(x, f32), f32(88.7))
    e = np.exp(x.astype(np.float64)).astype(f32)
    return (f32(1.0) / ((e + f32(1.0)) + f32(1e-16))).astype(f32)


def _element(objective, y, p, huber_slope):
    """(g, h) before the weight, float32, element-wise."""
    with np.errstate(all="ignore"):
        if objective == "reg:squarederror":
            return (p - y).astype(f32), np.ones_like(y, f32)
        if objective == "reg:pseudohubererror":
            s = f32(huber_slope)
            s2 = f32(s * s)
            z = (p - y).astype(f32)
            scale_sqrt = np.sqrt(f32(1.0) + (z * z) / s2).astype(f32)
            return (z / scale_sqrt).astype(f32), (s2 / ((s2 + z * z) * scale_sqrt)).astype(f32)
        if objective == "reg:squaredlogerror":
            p = np.maximum(p, f32(-1.0 + 1e-6))
            lp = np.log1p(p.astype(np.float64)).astype(f32)
            ly = np.log1p(y.astype(np.float64)).astype(f32)
            g = ((lp - ly) / (p + f32(1.0))).astype(f32)
            h = np.maximum((-lp + ly + f32(1.0)) / ((p + f32(1.0)) * (p + f32(1.0))), f32(1e-6)).astype(f32)
            return g, h
        if objective in LOGISTIC:
            q = sigmoid(p)
            return (q - y).astype(f32), np.maximum(q * (f32(1.0) - q), f32(1e-16)).astype(f32)
    raise ValueError("not a multi-target objective: %s" % objective)


def gradient(objective, margin, Y, weight=None, scale_pos_weight=1.0, huber_slope=1.0, keep=None):
    """float32 (n, T, 2): every element's (g, h); rows outside `keep` (the row sample, shared by the targets) get (0, 0)."""
    Y = np.asarray(Y, f32)
    n, T = Y.shape
    m = np.zeros((n, T), f32) if margin is None else np.asarray(margin, f32).reshape(n, T)
    w = np.ones(n, f32) if weight is None else np.asarray(weight, f32)
    out = np.zeros((n, T, 2), f32)
    for j in range(T):
        y = Y[:, j]
        if objective == "reg:absoluteerror":
            gp = AR.gradient(m[:, j], y, weight, keep)
            out[:, j] = gp
            continue
        wj = np.where(y == f32(1.0), (w * f32(scale_pos_weight)).astype(f32), w)
        g, h = _element(objective, y, m[:, j], huber_slope)
        g, h = (g * wj).astype(f32), (h * wj).astype(f32)
        if keep is not None:
            g[~keep] = 0
            h[~keep] = 0
        out[:, j, 0], out[:, j, 1] = g, h
    return out


def target_absmax(gp):
    """(T, 2) float32: each target's max|g| and max h (the fixed-point grid of its trees)."""
    gp = np.asarray(gp, f32)
    return np.stack([np.abs(gp[:, :, 0]).max(axis=0), gp[:, :, 1].max(axis=0)], axis=1).astype(f32)


def intercept(objective, Y, weight=None, scale_pos_weight=1.0, huber_slope=1.0):
    """The estimated base_score of a model trained on Y (n, T) without base_score (float32)."""
    Y = np.asarray(Y, f32)
    T = Y.shape[1]
    if objective == "reg:absoluteerror":
        total = 0.0
        for j in range(T):
            total += float(AR.base_score(Y[:, j], weight))
        return f32(total / T)
    gp = gradient(objective, None, Y, weight, scale_pos_weight, huber_slope)
    total = 0.0
    for j in range(T):
        G, H = gp[:, j, 0].astype(np.float64).sum(), gp[:, j, 1].astype(np.float64).sum()
        total += float(f32(0.0) if H <= 0 else f32(-G / H))
    w = f32(total / T)
    if objective in LOGISTIC:
        x = min(-w, f32(88.7))
        return f32(f32(1.0) / (f32(np.exp(np.float64(x))) + f32(1.0) + f32(1e-16)))
    return w


def _loss(metric, y, p, threshold, huber_slope):
    with np.errstate(all="ignore"):
        if metric == "rmse":
            return (p - y) ** 2
        if metric == "rmsle":
            return (np.log1p(y) - np.log1p(p)) ** 2
        if metric == "mae":
            return np.abs(p - y)
        if metric == "mape":
            return np.abs((y - p) / y)
        if metric == "mphe":
            z = (y - p) / huber_slope
            return huber_slope ** 2 * (np.sqrt(1.0 + z * z) - 1.0)
        if metric == "logloss":
            eps = 1e-16
            pc = np.clip(p, eps, 1.0 - eps)
            return -y * np.log(pc) - (1.0 - y) * np.log(1.0 - pc)
        if metric == "error":
            return np.where(p > threshold, 1.0 - y, y)
    raise ValueError("not an element-wise metric: %s" % metric)


def metric(name, Y, pred, weight=None, huber_slope=1.0):
    """The value of element-wise metric `name` (error@t included) on predictions pred (n, T) after the transform, in double."""
    Y = np.asarray(Y, np.float64)
    n, T = Y.shape
    p = np.asarray(pred, np.float64).reshape(n, T)
    w = np.ones(n) if weight is None else np.asarray(weight, np.float64)
    base, threshold = name, 0.5
    if name.startswith("error@"):
        base, threshold = "error", float(name[6:])
    loss = _loss(base, Y, p, threshold, huber_slope)
    v = float((loss * w[:, None]).sum() / (T * w.sum()))
    return float(np.sqrt(v)) if base in ("rmse", "rmsle") else v


def shapes(n, T, F, trees):
    """What predict() returns for a T-target model with `trees` trees over F features."""
    return {"value": (n, T), "margin": (n, T), "strict_shape": (n, T), "pred_leaf": (n, trees), "pred_contribs": (n, T, F + 1)}
