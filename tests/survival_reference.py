"""Host restatement of the survival objectives and metrics (survival:aft, survival:cox) -- TEST INFRASTRUCTURE.

The gradients restate upstream xgboost as it writes them [UPSTREAM-RECALL: src/common/survival_util.h, src/objective/aft_obj.cu,
src/objective/regression_obj.cu CoxRegression::GetGradient, src/metric/survival_metric.cu, elementwise_metric.cu EvalCox]:
AFT element-wise in float64, Cox as one sequential float64 loop with upstream's running subtraction of the risk-set sums.
`SurvivalTrainer` grows the trees with the oracle's trainer (oracle/gbt_oracle.py, unchanged): each round it hands the oracle
squared-error carrier labels and weights whose gradient pairs are the survival pairs (hessians exactly, gradients exactly or
to one ulp, see `carrier`), with the margins at zero, so the oracle's splits, leaves and fixed-point grid see the survival
gradients.
"""
import math

import numpy as np
from scipy import special

from split_reference import rng_uniform

f32 = np.float32
DISTS = {"normal": 0, "logistic": 1, "extreme": 2}
MIN_G, MAX_G, MIN_H, MAX_H, EPS = -15.0, 15.0, 1e-16, 15.0, 1e-12
UNC, RIGHT, LEFT, INTERVAL = 0, 1, 2, 3


# ---- AFT distributions of z = (ln y - m) / sigma, float64, in the order upstream writes the expressions.
# _JITTER = (relative size, bit): when set, every exp() / erf() result is moved by that relative amount, up or down by bit `bit`
# of its argument; `aft_conditioned` uses it to find the rows whose float32 pairs depend on the last bits of the math library.
_JITTER = (0.0, 0)


def _jit(v, x):
    j, bit = _JITTER
    if j == 0.0:
        return v
    b = np.ascontiguousarray(np.asarray(x, np.float64)).view(np.uint64)
    sgn = np.where((b >> np.uint64(bit)) & np.uint64(1), 1.0, -1.0)
    return v * (1.0 + j * sgn)


def _exp(x):
    return _jit(np.exp(x), x)


def _erf(x):
    return _jit(special.erf(x), x)


def pdf(d, z):
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        if d == 0:
            return _exp(-z * z / 2.0) / math.sqrt(2.0 * 3.14159265358979323846)
        w = _exp(z)
        if d == 1:
            sd = 1.0 + w
            return np.where(np.isinf(w) | np.isinf(w * w), 0.0, w / (sd * sd))
        return np.where(np.isinf(w), 0.0, w * _exp(-w))


def cdf(d, z):
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        if d == 0:
            return 0.5 * (1.0 + _erf(z / math.sqrt(2.0)))
        w = _exp(z)
        if d == 1:
            return np.where(np.isinf(w), 1.0, w / (1.0 + w))
        return 1.0 - _exp(-w)


def grad_pdf(d, z):
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        if d == 0:
            return -z * pdf(d, z)
        w = _exp(z)
        if d == 1:
            return np.where(np.isinf(w), 0.0, pdf(d, z) * (1.0 - w) / (1.0 + w))
        return np.where(np.isinf(w), 0.0, (1.0 - w) * pdf(d, z))


def hess_pdf(d, z):
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        if d == 0:
            return (z * z - 1.0) * pdf(d, z)
        w = _exp(z)
        bad = np.isinf(w) | np.isinf(w * w)
        if d == 1:
            return np.where(bad, 0.0, pdf(d, z) * (w * w - 4.0 * w + 1.0) / ((1.0 + w) * (1.0 + w)))
        return np.where(bad, 0.0, (w * w - 3.0 * w + 1.0) * pdf(d, z))


# limits at an infinite prediction [UPSTREAM-RECALL: GetLimitGradAtInfPred / GetLimitHessAtInfPred]; sign = z > 0
def limit_grad(d, c, sign, s):
    if d == 0:
        tab = {UNC: (MIN_G, MAX_G), INTERVAL: (MIN_G, MAX_G), RIGHT: (MIN_G, 0.0), LEFT: (0.0, MAX_G)}
    elif d == 1:
        tab = {UNC: (-1.0 / s, 1.0 / s), INTERVAL: (-1.0 / s, 1.0 / s), RIGHT: (-1.0 / s, 0.0), LEFT: (0.0, 1.0 / s)}
    else:
        tab = {UNC: (MIN_G, 1.0 / s), INTERVAL: (MIN_G, 1.0 / s), RIGHT: (MIN_G, 0.0), LEFT: (0.0, 1.0 / s)}
    return tab[c][0] if sign else tab[c][1]


def limit_hess(d, c, sign, s):
    if d == 0:
        tab = {UNC: (1.0 / (s * s),) * 2, INTERVAL: (1.0 / (s * s),) * 2, RIGHT: (1.0 / (s * s), MIN_H), LEFT: (MIN_H, 1.0 / (s * s))}
    elif d == 1:
        tab = {c_: (MIN_H, MIN_H) for c_ in (UNC, RIGHT, LEFT, INTERVAL)}
    else:
        tab = {UNC: (MAX_H, MIN_H), INTERVAL: (MAX_H, MIN_H), RIGHT: (MAX_H, MIN_H), LEFT: (MIN_H, MIN_H)}
    return tab[c][0] if sign else tab[c][1]


def aft_grad_hess(dist, lower, upper, margin, sigma):
    """Clipped float64 (g, h) of the AFT negative log-likelihood per row (before weights)."""
    d = DISTS[dist] if isinstance(dist, str) else int(dist)
    yl = np.asarray(lower, np.float32).astype(np.float64)
    yu = np.asarray(upper, np.float32).astype(np.float64)
    m = np.asarray(margin, np.float32).astype(np.float64)
    s = float(np.float32(sigma))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lyl, lyu = np.log(yl), np.log(yu)
        unc = yl == yu
        right, left = np.isinf(yu), yl <= 0.0
        z = (lyl - m) / s
        zu = np.where(right, 0.0, (lyu - m) / s)
        zl = np.where(left, 0.0, (lyl - m) / s)
        p, gp, hp = pdf(d, z), grad_pdf(d, z), hess_pdf(d, z)
        pu = np.where(right, 0.0, pdf(d, zu)); cu = np.where(right, 1.0, cdf(d, zu)); gu = np.where(right, 0.0, grad_pdf(d, zu))
        pl = np.where(left, 0.0, pdf(d, zl)); cl = np.where(left, 0.0, cdf(d, zl)); gl = np.where(left, 0.0, grad_pdf(d, zl))
        cdiff, pdiff, gdiff = cu - cl, pu - pl, gu - gl
        sd = s * cdiff
        gnum = np.where(unc, gp, pdiff); gden = np.where(unc, s * p, s * cdiff)
        hnum = np.where(unc, -(p * hp - gp * gp), -(cdiff * gdiff - pdiff * pdiff)); hden = np.where(unc, s * s * p * p, sd * sd)
        g, h = gnum / gden, hnum / hden
    cens = np.where(unc, UNC, np.where(left, LEFT, np.where(right, RIGHT, INTERVAL)))
    sign = np.where(unc, z > 0.0, (zu > 0.0) | (zl > 0.0))
    for i in np.nonzero((gden < EPS) & ~np.isfinite(g))[0]:
        g[i] = limit_grad(d, int(cens[i]), bool(sign[i]), s)
    for i in np.nonzero((hden < EPS) & ~np.isfinite(h))[0]:
        h[i] = limit_hess(d, int(cens[i]), bool(sign[i]), s)
    return np.clip(g, MIN_G, MAX_G), np.clip(h, MIN_H, MAX_H)


def aft_conditioned(margin, lower, upper, weight=None, dist="normal", sigma=1.0, ulps=2):
    """Rows whose float32 (g * w, h * w) stay within `ulps` when every exp() / erf() result moves by about two double ulps
    (four patterns): outside them the pair depends on the last bits of the math library (cancellation in F_u - F_l, 1 + erf,
    f f'' - f'^2 far from the label), and two correct implementations of the same formula disagree there."""
    global _JITTER
    ref = aft_gradient(margin, lower, upper, weight, dist, sigma)
    ok = np.ones(len(ref), bool)
    try:
        for j, bit in ((4.5e-16, 0), (-4.5e-16, 0), (4.5e-16, 1), (-4.5e-16, 1)):
            _JITTER = (j, bit)
            alt = aft_gradient(margin, lower, upper, weight, dist, sigma)
            d = np.abs(ref.view(np.int32).astype(np.int64) - alt.view(np.int32).astype(np.int64)).max(axis=1)
            ok &= d <= ulps
    finally:
        _JITTER = (0.0, 0)
    return ok


def sample_mask(n, seed, rnd, subsample):
    """Rows the product keeps in round `rnd` (stream 0x2000 + round), as the gradient kernels draw them."""
    if subsample >= 1.0:
        return np.ones(n, bool)
    return rng_uniform(seed, 0x2000 + rnd, np.arange(n, dtype=np.uint64)) < f32(subsample)


def aft_gradient(margin, lower, upper, weight=None, dist="normal", sigma=1.0):
    """float32 (n, 2): (float(g) * w, float(h) * w) as upstream's AFTObj writes them."""
    g, h = aft_grad_hess(dist, lower, upper, margin, sigma)
    w = np.ones(len(g), np.float32) if weight is None else np.asarray(weight, np.float32)
    return np.stack([g.astype(np.float32) * w, h.astype(np.float32) * w], axis=1)


def cox_gradient(margin, y, weight=None, float_total=True):
    """Upstream's CoxRegression::GetGradient, sequential: float32 (n, 2).  The total starts as a double sum of float exp() in
    sorted order (float_total=False: of double exp()); each later tie group subtracts the accumulated double exp() of the groups
    before it (Breslow).  The float total leaves its rounding in every D: near the end of the order, where D is a handful of
    rows, that is a relative error of up to a few percent on millions of rows."""
    m = np.asarray(margin, np.float32).reshape(-1)
    y = np.asarray(y, np.float32)
    n = len(m)
    w = np.ones(n, np.float32) if weight is None else np.asarray(weight, np.float32)
    order = np.argsort(np.abs(y), kind="stable")
    ef = np.exp(m[order]).astype(np.float64) if float_total else np.exp(m[order].astype(np.float64))   # std::exp(float) upstream
    exp_p_sum = 0.0
    for v in ef.tolist():
        exp_p_sum += v
    out = np.zeros((n, 2), np.float32)
    ml, yl, wl = m.astype(np.float64).tolist(), y.astype(np.float64).tolist(), w.astype(np.float64).tolist()
    r_k = s_k = last_exp_p = last_abs_y = acc = 0.0
    gs, hs = np.zeros(n), np.zeros(n)
    for ind in order.tolist():
        exp_p = math.exp(ml[ind]); yv = yl[ind]; abs_y = abs(yv)
        acc += last_exp_p
        if last_abs_y < abs_y:
            exp_p_sum -= acc
            acc = 0.0
        if yv > 0:
            r_k += 1.0 / exp_p_sum
            s_k += 1.0 / (exp_p_sum * exp_p_sum)
        gs[ind] = (exp_p * r_k - (1.0 if yv > 0 else 0.0)) * wl[ind]
        hs[ind] = (exp_p * r_k - exp_p * exp_p * s_k) * wl[ind]
        last_abs_y = abs_y; last_exp_p = exp_p
    out[:, 0] = gs.astype(np.float32); out[:, 1] = hs.astype(np.float32)
    return out


def gradient(params, margin, label=None, lower=None, upper=None, weight=None, rnd=0):
    """The survival objective of `params` at `margin` with round `rnd`'s row sample: float32 (n, 2)."""
    obj = params["objective"]
    if obj == "survival:aft":
        gp = aft_gradient(margin, lower, upper, weight, params.get("aft_loss_distribution", "normal"),
                          float(params.get("aft_loss_distribution_scale", 1.0)))
    elif obj == "survival:cox":
        gp = cox_gradient(margin, label, weight)
    else:
        raise ValueError(obj)
    keep = sample_mask(len(gp), int(params.get("seed", 0)), rnd, float(params.get("subsample", 1.0)))
    gp[~keep] = 0.0
    return gp


# ---- metrics
def aft_nloglik(margin, lower, upper, weight=None, dist="normal", sigma=1.0):
    d = DISTS[dist]
    yl = np.asarray(lower, np.float32).astype(np.float64)
    yu = np.asarray(upper, np.float32).astype(np.float64)
    m = np.asarray(margin, np.float32).astype(np.float64).reshape(-1)
    s = float(np.float32(sigma))
    w = np.ones(len(m)) if weight is None else np.asarray(weight, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        unc = yl == yu
        z = (np.log(yl) - m) / s
        lu = -np.log(np.maximum(pdf(d, z) / (s * yl), EPS))
        cu = np.where(np.isinf(yu), 1.0, cdf(d, (np.log(yu) - m) / s))
        cl = np.where(yl <= 0.0, 0.0, cdf(d, (np.log(yl) - m) / s))
        lc = -np.log(np.maximum(cu - cl, EPS))
    return float(np.sum(np.where(unc, lu, lc) * w) / np.sum(w))


def interval_accuracy(margin, lower, upper, weight=None):
    p = np.exp(np.asarray(margin, np.float32).astype(np.float64).reshape(-1))
    yl = np.asarray(lower, np.float32).astype(np.float64)
    yu = np.asarray(upper, np.float32).astype(np.float64)
    w = np.ones(len(p)) if weight is None else np.asarray(weight, np.float32).astype(np.float64)
    return float(np.sum(((p >= yl) & (p <= yu)) * w) / np.sum(w))


def cox_nloglik(margin, y):
    """-sum over events of (m_i - ln D_i) / #events, D_i the exp(margin) sum over the rows with |y_j| >= |y_i|."""
    m = np.asarray(margin, np.float32).astype(np.float64).reshape(-1)
    a = np.abs(np.asarray(y, np.float32))
    order = np.argsort(a, kind="stable")
    e = np.exp(m[order])
    suf = np.cumsum(e[::-1])[::-1]
    first = np.searchsorted(a[order], a[order], side="left")       # tie-group head of each sorted position
    ev = np.asarray(y, np.float32)[order] > 0
    return float(-np.sum(m[order][ev] - np.log(suf[first][ev])) / ev.sum())


# ---- trees: the oracle's trainer on squared-error carriers of the survival gradient pairs
def carrier(gp):
    """Labels y' and weights w' for reg:squarederror at margin 0: fl(1 * w') == h exactly, and fl(fl(0 - y') * w') == g where a
    float32 y' reaches g (about nine rows in ten when h > 1), else the nearest float32 to g (one ulp away).  The fixed-point
    grid of the histograms absorbs that ulp except on rounding ties, so trees compare by structure and leaf tolerance."""
    g, h = gp[:, 0].astype(np.float32), gp[:, 1].astype(np.float32)
    zero = h == 0
    assert np.all(g[zero] == 0), "a zero hessian with a non-zero gradient has no carrier"
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        x0 = np.where(zero, f32(0), (g.astype(np.float64) / np.where(zero, 1.0, h).astype(np.float64)).astype(np.float32))
        best, err = x0.copy(), np.abs((x0 * h).astype(np.float64) - g)
        for step in (1, 2):
            for to in (f32(np.inf), f32(-np.inf)):
                cand = x0
                for _ in range(step):
                    cand = np.nextafter(cand, to)
                e = np.abs((cand * h).astype(np.float64) - g)
                better = ~zero & (e < err)
                best[better], err[better] = cand[better], e[better]
    return (-best).astype(np.float32), h.copy()


class SurvivalTrainer:
    """One boosting round per update(): the product's survival gradients (this module) at the current margins, the tree grown
    by the oracle from their carriers, the margins advanced in fp32 by its leaves."""

    def __init__(self, params, X, label=None, lower=None, upper=None, weight=None, bins=None, cuts=None, device_grid=True):
        from oracle import gbt_oracle as O
        self.params = dict(params)
        n = len(X)
        self.label, self.lower, self.upper, self.weight = label, lower, upper, weight
        op = {k: v for k, v in params.items() if k not in ("objective", "subsample", "aft_loss_distribution", "aft_loss_distribution_scale",
                                                              "eval_metric")}
        op.update(objective="reg:squarederror", base_score=0.5)
        self._y = np.zeros(n, np.float32)
        self._w = np.ones(n, np.float32)
        self.t = O.Trainer(op, X=X, y=self._y, weights=self._w, bins=bins, cuts=cuts, base_score=0.5)
        if device_grid:
            self.t.set_device_grid()
        self.m = np.full(n, np.log(f32(float(params.get("base_score", 0.5)))), np.float32)
        self.rounds = 0

    def update(self):
        gp = gradient(self.params, self.m, self.label, self.lower, self.upper, self.weight, self.rounds)
        y, w = carrier(gp)
        self.t.y[:] = y
        self.t.w[:] = w
        self.t.set_margins(np.zeros(len(y), np.float32))
        self.t.update()
        self.m = (self.m + self.t.margins()[:, 0]).astype(np.float32)
        self.rounds += 1

    def model(self):
        return self.t.model()

    def margins(self):
        return self.m.reshape(-1, 1)
