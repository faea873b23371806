"""Split evaluation and node expansion of one node, restated in NumPy from upstream xgboost's rules (the CPU hist updater's
EnumerateSplit, SplitEntry::NeedReplace, ExpandEntry::IsValid and TreeEvaluator) in the float / double mix of
oracle/gbt_oracle.c: statistics and weights in float64, weights rounded to float32, the max_delta_step / monotone gain
-(2 g w + (h + lambda) w^2) in float32 with every operation rounded on its own (no fused multiply-add).

The inputs are the device's: an int64 fixed-point histogram per feature and bin, the node totals in grid units, and the
grid's power-of-two scales, which dequantise exactly (int64 * 2^-k in float64).  Every function is vectorised over all
candidates of all features, so that wide layouts (tens of thousands of features) stay cheap.
"""
import numpy as np

f32 = np.float32
K_RT_EPS = f32(1e-6)


# ------------------------------------------------------------------------------------------------ grid
def grad_bits_for(n):
    """Magnitude bits of the fixed-point g (csrc/engine.h grad_bits_for): 21 up to 2^20 rows, 18 above."""
    return 21 if n <= (1 << 20) else 18


def scales_for(max_g, max_h, grad_bits):
    """[sg, sh, 1/sg, 1/sh] as float32: g on a 2^(bits - eg) grid, h on a 2^(bits + 1 - eh) grid, m < 2^e."""
    def exp_of(m):
        m = f32(m)
        return int(np.frexp(m)[1]) if (m > 0 and np.isfinite(m)) else 0
    sg = f32(np.ldexp(1.0, grad_bits - exp_of(max_g)))
    sh = f32(np.ldexp(1.0, grad_bits + 1 - exp_of(max_h)))
    return np.array([sg, sh, f32(1) / sg, f32(1) / sh], np.float32)


# ------------------------------------------------------------------------------------------------ split arithmetic
class Params:
    def __init__(self, eta=0.3, reg_lambda=1.0, alpha=0.0, gamma=0.0, min_child_weight=1.0, max_delta_step=0.0, max_depth=6):
        self.eta, self.lam, self.alpha, self.gamma = f32(eta), f32(reg_lambda), f32(alpha), f32(gamma)
        self.mcw, self.mds, self.max_depth = f32(min_child_weight), f32(max_delta_step), int(max_depth)

    @classmethod
    def of(cls, params):
        g = params.get
        return cls(eta=g("eta", 0.3), reg_lambda=g("lambda", g("reg_lambda", 1.0)), alpha=g("alpha", 0.0), gamma=g("gamma", 0.0),
                   min_child_weight=g("min_child_weight", 1.0), max_delta_step=g("max_delta_step", 0.0), max_depth=g("max_depth", 6))


def threshold_l1(w, alpha):
    w = np.asarray(w, np.float64)
    a = float(alpha)
    return np.where(w > a, w - a, np.where(w < -a, w + a, 0.0))


def calc_weight(p, G, H):
    """-T(G) / (H + lambda) in float64, clipped to +-max_delta_step, rounded to float32; 0 below min_child_weight."""
    G = np.asarray(G, np.float64); H = np.asarray(H, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        dw = -threshold_l1(G, p.alpha) / (H + float(p.lam))
    if p.mds != 0:
        dw = np.where(np.abs(dw) > float(p.mds), np.copysign(float(p.mds), dw), dw)
    return np.where((H < float(p.mcw)) | (H <= 0.0), f32(0), dw.astype(np.float32)).astype(np.float32)


def gain_at_weight(p, G, H, w):
    """-(2 g w + (h + lambda) w^2) in float32, each operation rounded separately; 0 for an empty hessian."""
    g = np.asarray(G, np.float64).astype(np.float32); h = np.asarray(H, np.float64).astype(np.float32); w = np.asarray(w, np.float32)
    two_gw = (f32(2) * g) * w
    hw2 = ((h + p.lam) * w) * w
    return np.where(np.asarray(H) <= 0.0, f32(0), -(two_gw + hw2)).astype(np.float32)


def calc_gain_given_weight(p, G, H, w):
    if p.mds == 0:
        G = np.asarray(G, np.float64); H = np.asarray(H, np.float64)
        t = threshold_l1(G, p.alpha)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = (t * t / (H + float(p.lam))).astype(np.float32)
        return np.where(H <= 0.0, f32(0), v).astype(np.float32)
    return gain_at_weight(p, G, H, w)


def calc_gain(p, G, H):
    return calc_gain_given_weight(p, G, H, calc_weight(p, G, H))


# ------------------------------------------------------------------------------------------------ colsample_bynode
_M64 = (1 << 64) - 1


def _splitmix64(x):
    x = x.astype(np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def rng_uniform(seed, stream, idx):
    """csrc/rng.h: splitmix64(splitmix64((seed << 32) ^ stream) ^ idx), top 24 bits as a float32 in [0, 1)."""
    inner = _splitmix64(np.array([((int(seed) << 32) ^ int(stream)) & _M64], np.uint64))[0]
    h = _splitmix64(np.asarray(idx, np.uint64) ^ inner)
    return (h >> np.uint64(40)).astype(np.float32) * f32(1.0 / 16777216.0)


def bynode_mask(parent, frac, seed, tree_index, nid):
    """The node's column subset inside `parent`: the max(1, floor(frac * |parent|)) features with the smallest draw, ties to
    the lower index (upstream ColumnSampler semantics with the project's counter-based draw)."""
    parent = np.asarray(parent, bool)
    if frac >= 1.0:
        return parent.copy()
    F = len(parent)
    stream = 0x80000000 + (int(tree_index) << 20) + int(nid)
    u = rng_uniform(seed, stream, np.arange(F, dtype=np.uint64))
    idx = np.flatnonzero(parent)
    keep = max(1, int(np.floor(f32(frac) * f32(len(idx)))))
    order = idx[np.lexsort((idx, u[idx]))]
    m = np.zeros(F, bool)
    m[order[:keep]] = True
    return m


# ------------------------------------------------------------------------------------------------ test nodes
def synth_node(rng, nbins, n_rows=400, missing_frac=0.0, gmax=1 << 21, hmax=1 << 22, dup=()):
    """An exact int64 histogram [F][256][2] of synthetic quantised rows (bin per feature, -1 = missing; g_q, h_q >= 0), the node
    totals, and cuts (cut_ptrs, increasing cut_vals, min_vals).  dup: (src, dst) pairs, column dst is a copy of column src."""
    nbins = np.asarray(nbins, np.int64)
    F = len(nbins)
    bins = (rng.random((n_rows, F)) * nbins).astype(np.int64)
    if missing_frac > 0:
        bins[rng.random((n_rows, F)) < missing_frac] = -1
    for s, d in dup:
        bins[:, d] = bins[:, s]
    gq = rng.integers(-gmax, gmax + 1, n_rows, dtype=np.int64)
    hq = rng.integers(0, hmax + 1, n_rows, dtype=np.int64)
    hist = np.zeros((F, 256, 2), np.int64)
    for f in range(F):
        m = bins[:, f] >= 0
        np.add.at(hist[f, :, 0], bins[m, f], gq[m])
        np.add.at(hist[f, :, 1], bins[m, f], hq[m])
    cut_ptrs = np.concatenate([[0], np.cumsum(nbins)]).astype(np.int32)
    cut_vals = np.concatenate([f + 0.25 * np.arange(1, k + 1) for f, k in enumerate(nbins)]).astype(np.float32)
    min_vals = np.arange(F, dtype=np.float32)
    return hist, (int(gq.sum()), int(hq.sum())), (cut_ptrs, cut_vals, min_vals)


# ------------------------------------------------------------------------------------------------ one node
def _cands(p, hist, cut_ptrs, has_missing, tot, isg, ish, lo, hi, mono, usable, root_gain):
    """Every candidate of every usable feature: (feature, bin, dleft, ord, GLq, HLq, loss) arrays; loss NaN = not a candidate."""
    F = len(cut_ptrs) - 1
    nb = np.diff(cut_ptrs).astype(np.int64)
    feat = np.repeat(np.arange(F), nb)
    b = np.arange(int(cut_ptrs[F])) - np.repeat(cut_ptrs[:-1].astype(np.int64), nb)
    hg = hist[feat, b, 0].astype(np.int64); hh = hist[feat, b, 1].astype(np.int64)
    start = np.repeat(cut_ptrs[:-1].astype(np.int64), nb)
    cg = np.cumsum(hg); ch = np.cumsum(hh)
    off_g = np.concatenate([[0], cg])[start]; off_h = np.concatenate([[0], ch])[start]
    fwd_g = cg - off_g; fwd_h = ch - off_h                      # inclusive sums of bins <= b within the feature
    tG = np.zeros(F, np.int64); tH = np.zeros(F, np.int64)
    last = cut_ptrs[1:].astype(np.int64) - 1
    has = nb > 0
    tG[has] = fwd_g[last[has]]; tH[has] = fwd_h[last[has]]
    Gq, Hq = int(tot[0]), int(tot[1])
    fmiss = has_missing & ((tG != Gq) | (tH != Hq))
    # forward: missing right; backward: missing left, right = bins >= b
    bwd_rg = tG[feat] - (fwd_g - hg); bwd_rh = tH[feat] - (fwd_h - hh)
    out = []
    for dleft in (0, 1):
        if dleft == 0:
            GLq, HLq = fwd_g, fwd_h
            sel = usable[feat]
            ordv = b
            binv = b
        else:
            GLq, HLq = Gq - bwd_rg, Hq - bwd_rh
            sel = usable[feat] & fmiss[feat]
            ordv = 256 + (255 - b)
            binv = b - 1
        GRq, HRq = Gq - GLq, Hq - HLq
        GL, HL, GR, HR = GLq * isg, HLq * ish, GRq * isg, HRq * ish
        ok = sel & (HL >= float(p.mcw)) & (HR >= float(p.mcw))
        if mono is None:
            gsum = calc_gain_given_weight(p, GL, HL, calc_weight(p, GL, HL)) + calc_gain_given_weight(p, GR, HR, calc_weight(p, GR, HR))
        else:
            wl = np.clip(calc_weight(p, GL, HL), lo, hi).astype(np.float32)
            wr = np.clip(calc_weight(p, GR, HR), lo, hi).astype(np.float32)
            c = np.asarray(mono)[feat]
            ok &= (c == 0) | ((c > 0) & (wl <= wr)) | ((c < 0) & (wl >= wr))
            gsum = gain_at_weight(p, GL, HL, wl) + gain_at_weight(p, GR, HR, wr)
        loss = (gsum.astype(np.float32) - f32(root_gain)).astype(np.float32)
        loss = np.where(ok, loss, np.nan).astype(np.float32)
        out.append((feat, binv, np.full(len(feat), dleft), ordv, GLq, HLq, loss))
    return [np.concatenate(x) for x in zip(*out)]


def eval_node(params, hist, cut_ptrs, cut_vals, min_vals, has_missing, tot, scales, lower=-np.inf, upper=np.inf, monotone=None,
              feat_mask=None, colsample_bynode=1.0, seed=0, tree_index=0, nid=0):
    """Split evaluation + expansion of a root (max_depth >= 1): the fields XGB200BoosterEvalRootSplit reports, floats as float32."""
    p = params if isinstance(params, Params) else Params.of(params)
    hist = np.asarray(hist, np.int64)
    cut_ptrs = np.asarray(cut_ptrs, np.int64)
    F = len(cut_ptrs) - 1
    isg, ish = float(scales[2]), float(scales[3])
    G, H = int(tot[0]) * isg, int(tot[1]) * ish
    lo, hi = f32(lower), f32(upper)
    mono = None if monotone is None or not np.any(monotone) else np.asarray(list(monotone) + [0] * (F - len(monotone)), np.int64)
    usable = np.ones(F, bool) if feat_mask is None else np.asarray(feat_mask, bool)
    if feat_mask is not None or colsample_bynode < 1.0:
        usable = bynode_mask(usable, colsample_bynode, seed, tree_index, nid)
    w = calc_weight(p, G, H)[()]
    if mono is not None:
        w = np.clip(w, lo, hi).astype(np.float32)[()]
    root_gain = gain_at_weight(p, G, H, w)[()] if mono is not None else calc_gain(p, G, H)[()]
    feat, binv, dleft, ordv, GLq, HLq, loss = _cands(p, hist, cut_ptrs, bool(has_missing), tot, isg, ish, lo, hi, mono, usable, root_gain)
    # SplitEntry::NeedReplace: larger loss_chg; a tie goes to the lower feature, then to the earlier candidate in scan order
    cand = np.flatnonzero(np.isfinite(loss) & (loss > 0))
    best = None
    if len(cand):
        top = cand[loss[cand] == loss[cand].max()]
        top = top[feat[top] == feat[top].min()]
        i = top[np.argmin(ordv[top])]
        best = dict(loss_chg=f32(loss[i]), feature=int(feat[i]), bin=int(binv[i]), dleft=int(dleft[i]), ord=int(ordv[i]), GL=int(GLq[i]), HL=int(HLq[i]))
    res = dict(root_gain=f32(root_gain), weight=f32(w), best=best)
    # ExpandEntry::IsValid (+ Driver::Push for loss-guided growth: the same eps)
    valid = best is not None and best["loss_chg"] > K_RT_EPS and best["HL"] != 0 and int(tot[1]) - best["HL"] != 0 \
        and not (best["loss_chg"] < p.gamma)
    res["expanded"] = bool(valid)
    sum_hess = f32(H)
    if not valid:
        res["tree"] = dict(left=[-1], right=[-1], parent=[2147483647], split_index=[0], split_bin=[-1], default_left=[0],
                           split_cond=[f32(p.eta * f32(w))], base_weight=[f32(w)], loss_chg=[f32(0)], sum_hess=[sum_hess])
        res["children"] = []
        return res
    f = best["feature"]
    GLq, HLq = best["GL"], best["HL"]
    GRq, HRq = int(tot[0]) - GLq, int(tot[1]) - HLq
    GL, HL, GR, HR = GLq * isg, HLq * ish, GRq * isg, HRq * ish
    wl, wr = calc_weight(p, GL, HL)[()], calc_weight(p, GR, HR)[()]
    bounds = [(lo, hi), (lo, hi)]
    if mono is not None:
        wl, wr = np.clip(wl, lo, hi).astype(np.float32)[()], np.clip(wr, lo, hi).astype(np.float32)[()]
        mid = f32((f32(wl) + f32(wr)) / f32(2))
        if mono[f] < 0:
            bounds = [(mid, hi), (lo, mid)]
        elif mono[f] > 0:
            bounds = [(lo, mid), (mid, hi)]
    cb = int(cut_ptrs[f])
    thr = f32(min_vals[f]) if (best["dleft"] and best["bin"] < 0) else f32(cut_vals[cb + best["bin"]])
    lw, rw = f32(p.eta * f32(wl)), f32(p.eta * f32(wr))
    res["tree"] = dict(left=[1, -1, -1], right=[2, -1, -1], parent=[2147483647, 0, 0], split_index=[f, 0, 0], split_bin=[best["bin"], -1, -1],
                       default_left=[best["dleft"], 0, 0], split_cond=[thr, lw, rw], base_weight=[f32(w), lw, rw],
                       loss_chg=[best["loss_chg"], f32(0), f32(0)], sum_hess=[sum_hess, f32(HL), f32(HR)])
    res["children"] = [dict(G=GLq, H=HLq, lower=bounds[0][0], upper=bounds[0][1]), dict(G=GRq, H=HRq, lower=bounds[1][0], upper=bounds[1][1])]
    return res
