"""Host restatement of sampling_method=gradient_based -- TEST INFRASTRUCTURE.

Upstream semantics [UPSTREAM-RECALL: xgboost 3.0.5 src/tree/gpu_hist/gradient_based_sampler.cu GradientBasedSampler,
minimal-variance sampling]: only with subsample < 1; per tree, rag = sqrtf(g^2 + lambda h^2) with the sampler's own
lambda = 0.1, k = (size_t)(n * subsample) computed in float, the threshold u with sum_i min(1, rag_i / u) = k, and each row
with p = rag / u < 1 kept with probability p as (g / p, h / p); rows with p >= 1 kept as they are.

The product's rule, restated exactly here (csrc/sampling.cu):
- k = max(1, int(float32(n) * float32(subsample)));
- u from a radix descent over the uint32 bits of rag (non-finite rag keyed as +inf), 8 bits per pass: each pass counts the rows
  and sums rag_q = rint(rag * 2^(bits - e)) per digit (int64; every value of the bucket below 2^e, e from its largest key,
  bits = grad_bits_for(n)), evaluates phi(v) = S_lt + v * (N_ge - k) in double at every finite bucket edge, S_lt adding the
  buckets' sums times 2^(e - bits) in bucket order, and descends into the last bucket with phi > 0; finally
  u = fl32(S_below / (k - N_above)), or next(x) when that quotient is undefined, or 0 (every row kept as is) when no edge had
  phi > 0, i.e. when k >= the rows with rag > 0;
- the keep draw of row r is split_reference.rng_uniform(seed, stream, r + row_offset), the stream of the round's uniform sample
  (forest_reference.row_stream), one draw per row shared by the classes;
- non-finite rag: kept as is.

`upstream_threshold` is upstream's float sort-and-scan rule, and `brute_threshold` an O(n^2) solve in float64, for comparison.
`GbsTrainer` hands the sampled pairs to the unchanged oracle trainer through carrier labels and weights
(survival_reference.carrier), `GbsAbsErrorTrainer` does so for reg:absoluteerror (absoluteerror_reference)."""
import math

import numpy as np

from split_reference import grad_bits_for, rng_uniform

f32 = np.float32
LAMBDA = f32(0.1)          # the sampler's constant [UPSTREAM-RECALL], csrc/sampling.h kGbsLambda
DIGIT_BITS, BUCKETS, PASSES = 8, 256, 4
INF_KEY = 0x7F800000


def rag(gp):
    """float32 sqrt(g^2 + lambda h^2), every operation rounded on its own."""
    gp = np.asarray(gp, np.float32)
    g, h = gp[..., 0], gp[..., 1]
    with np.errstate(over="ignore", invalid="ignore"):
        return np.sqrt(g * g + LAMBDA * (h * h)).astype(np.float32)


def target(n, subsample):
    return max(1, int(f32(n) * f32(subsample)))


def _keys(x):
    k = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.int64)
    k[~np.isfinite(x)] = INF_KEY
    return k


def grid_exp(lo, shift, bits):
    """The grid exponent of the bucket of keys [lo, lo + 2^shift): bits - e, every value below 2^e (e = 128 where the bucket
    reaches the non-finite keys), capped at 126."""
    top = lo + (1 << shift) - 1
    e = 128
    if top < INF_KEY:
        m = np.array([top], np.uint32).view(np.float32)[0]
        e = int(np.frexp(m)[1]) if m > 0 else 0
    return min(bits - e, 126)


def threshold(r, subsample):
    """The product's u for one column of rag values r (float32)."""
    r = np.asarray(r, np.float32)
    n = len(r)
    k_t = target(n, subsample)
    bits = grad_bits_for(n)
    fin = np.isfinite(r)
    rf = np.where(fin, r, f32(0)).astype(np.float32)
    key = _keys(r)
    prefix, s_lo, n_hi = 0, 0.0, 0
    for p in range(PASSES):
        shift = 32 - DIGIT_BITS * (p + 1)
        hi_mask = 0 if p == 0 else (0xFFFFFFFF << (shift + DIGIT_BITS)) & 0xFFFFFFFF
        sel = (key & hi_mask) == prefix
        digit = (key[sel] >> shift) & (BUCKETS - 1)
        ex = np.array([grid_exp(prefix | (b << shift), shift, bits) for b in range(BUCKETS)])
        scale = np.ldexp(np.ones(BUCKETS, np.float32), ex).astype(np.float32)
        with np.errstate(over="ignore", invalid="ignore"):
            q = np.rint(rf[sel] * scale[digit]).astype(np.int64)
        cnt = np.bincount(digit, minlength=BUCKETS).astype(np.int64)
        sm = np.zeros(BUCKETS, np.int64)
        np.add.at(sm, digit, q)
        total = int(cnt.sum())
        pick, s_lt, n_ge, s_pick, n_pick = 0, s_lo, n_hi + total, s_lo, n_hi + total
        for b in range(BUCKETS):
            edge = prefix | (b << shift)
            if edge >= INF_KEY:
                break
            v = float(np.array([edge], np.uint32).view(np.float32)[0])
            phi = s_lt + v * float(n_ge - k_t)
            if phi > 0.0:
                pick, s_pick, n_pick = b, s_lt, n_ge
            s_lt = s_lt + math.ldexp(float(sm[b]), -int(ex[b]))
            n_ge -= int(cnt[b])
        s_bucket = math.ldexp(float(sm[pick]), -int(ex[pick]))
        prefix |= pick << shift
        s_lo, n_hi = s_pick, n_pick - int(cnt[pick])
        if p == PASSES - 1:
            if prefix == 0:
                return f32(0)
            s_below, den = s_lo + s_bucket, k_t - n_hi
            if s_below > 0 and den > 0:
                return f32(s_below / float(den))
            return np.array([prefix + 1], np.uint32).view(np.float32)[0]


def sample(gp, u, draw):
    """One column's pairs gp (n, 2) kept by threshold u with the per-row draws: what the sampling kernel writes."""
    gp = np.asarray(gp, np.float32)
    out = gp.copy()
    if u == 0:
        return out
    r = rag(gp)
    fin = np.isfinite(r)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        p = np.where(fin, r, f32(0)) / f32(u)
        scaled = fin & (p < 1)
        keep = scaled & (draw < p)
        out[scaled & ~keep] = 0
        out[keep, 0] = gp[keep, 0] / p[keep]
        out[keep, 1] = gp[keep, 1] / p[keep]
    return out.astype(np.float32)


def draws(seed, stream, n, row_offset=0):
    return rng_uniform(seed, stream, np.arange(n, dtype=np.uint64) + np.uint64(row_offset))


def gradient_based_sample(gp, subsample, seed=0, stream=0x2000, row_offset=0):
    """(u, sampled pairs) of one column: what XGB200GradientBasedSample returns."""
    gp = np.asarray(gp, np.float32)
    u = threshold(rag(gp), subsample)
    return u, sample(gp, u, draws(seed, stream, len(gp), row_offset))


def sample_classes(gp, subsample, seed, stream, row_offset=0):
    """gp (n, K, 2): every class on its own threshold, one draw per row shared by the classes (tree 0 of a round when stream is
    the round's uniform stream): what XGB200BoosterComputeGradient returns under gradient_based."""
    gp = np.asarray(gp, np.float32)
    d = draws(seed, stream, gp.shape[0], row_offset)
    out = np.empty_like(gp)
    for c in range(gp.shape[1]):
        out[:, c] = sample(gp[:, c], threshold(rag(gp[:, c]), subsample), d)
    return out


# ---- comparison rules
def upstream_threshold(r, subsample):
    """Upstream's float rule: sort ascending, append FLT_MAX, inclusive float scan S; the first i with
    rag_(i) < S_i / (k - n + i + 1) <= rag_(i+1) sets u (None when no index is valid)."""
    r = np.sort(np.asarray(r, np.float32))
    n = len(r)
    k = int(f32(n) * f32(subsample))
    a = np.append(r, f32(np.finfo(np.float32).max))
    S = np.cumsum(a, dtype=np.float32)
    for i in range(n):
        den = k - n + i + 1
        if den <= 0:
            continue
        u = f32(S[i] / f32(den))
        if a[i] < u <= a[i + 1]:
            return u
    return None


def brute_threshold(r, k):
    """The u > 0 with sum min(1, r / u) = k in float64 by trying every split of the sorted values: O(n^2)."""
    r = np.sort(np.asarray(r, np.float64))
    n = len(r)
    for above in range(n):
        den = k - above
        if den <= 0:
            break
        below = r[:n - above]
        u = sum(float(x) for x in below) / den
        lo = below[-1] if len(below) else 0.0
        hi = r[n - above] if above else np.inf
        if lo < u <= hi:
            return u
    return None


def kept_sum(r, u):
    """sum_i min(1, r_i / u) in float64."""
    r = np.asarray(r, np.float64)
    return float(np.sum(np.minimum(1.0, r / float(u))))


# ---- whole models on the oracle trainer
class GbsTrainer:
    """One boosting round per update() for a one-class objective, as csrc/booster.cu update_one_iter runs it under
    sampling_method=gradient_based: the round's unsampled pairs from grad_fn(margin, round) (the product's objective), one
    threshold per round, tree j of the round sampled with the draws of forest_reference.row_stream(round, j), grown by the
    oracle from the pairs' carriers at leaves fl(eta / P), margins advanced in float32.  booster=dart: the drop set and weights of
    tests/dart_reference.py, gradients at the margin without the dropped trees."""

    def __init__(self, params, X, grad_fn, m0, cuts=None, bins=None):
        from oracle import gbt_oracle as O
        from dart_reference import dart_param
        from forest_reference import forest_eta
        self.params = dict(params)
        self.X = np.ascontiguousarray(X, np.float32)
        n = len(self.X)
        self.grad_fn = grad_fn
        self.P = int(params.get("num_parallel_tree", 1))
        self.eta = float(params.get("eta", 0.3))
        self.dart = dart_param(params) if params.get("booster") == "dart" else None
        drop = ("objective", "subsample", "sampling_method", "eval_metric", "base_score", "num_parallel_tree", "booster", "rate_drop",
                "skip_drop", "one_drop", "sample_type", "normalize_type", "aft_loss_distribution", "aft_loss_distribution_scale")
        op = {k: v for k, v in params.items() if k not in drop}
        op.update(objective="reg:squarederror", base_score=0.5, eta=float(forest_eta(self.eta, self.P)))
        self.t = O.Trainer(op, X=self.X, y=np.zeros(n, np.float32), weights=np.ones(n, np.float32), cuts=cuts, bins=bins, base_score=0.5)
        self.t.set_device_grid()
        self.m = np.full(n, m0, np.float32)
        self.values = []                          # per tree: its leaf value on every row
        self.weights = []
        self.thresholds = []                      # per round
        self.exact = True                         # every carrier reproduced its pair bit for bit
        self.rounds = 0

    def update(self):
        from dart_reference import drop_set, normalisation
        from forest_reference import row_stream
        from survival_reference import carrier
        n = len(self.m)
        seed, rnd = int(self.params.get("seed", 0)), self.rounds
        sub = float(self.params["subsample"])
        w_new, m_grad = f32(1), self.m
        if self.dart is not None:
            D = drop_set(self.weights, rnd, seed, self.dart)
            factor, w_new = normalisation(len(D), self.eta, 1, self.dart["normalize_type"])
            m_grad = self.m.copy()
            for j in D:
                v, w = self.values[j], f32(self.weights[j])
                w2 = f32(w * factor)
                m_grad = m_grad - w * v
                self.m = self.m + f32(w2 - w) * v
                self.weights[j] = w2
        m_grad = np.asarray(m_grad, np.float32).copy()
        full = np.asarray(self.grad_fn(m_grad, rnd), np.float32).reshape(n, 2)
        u = threshold(rag(full), sub)
        self.thresholds.append(u)
        for j in range(self.P):
            gp = sample(full, u, draws(seed, row_stream(rnd, j), n))
            y, w = carrier(gp)
            self.exact &= bool(np.all(((f32(0) - y) * w).astype(np.float32) == gp[:, 0]))
            self.t.y[:] = y
            self.t.w[:] = w
            self.t.set_margins(np.zeros(n, np.float32))
            self.t.update()
            v = self.t.margins()[:, 0].astype(np.float32)
            self.values.append(v)
            self.m = (self.m + (v if self.dart is None else w_new * v)).astype(np.float32)
            self.weights.append(w_new)
        self.rounds += 1

    def model(self):
        return self.t.model()


def _absolute_error_trainer():
    from absoluteerror_reference import AbsErrorTrainer
    return AbsErrorTrainer


class GbsAbsErrorTrainer(_absolute_error_trainer()):
    """reg:absoluteerror under gradient_based (no dart): the round's pairs (sign(m - y) w, w) sampled per tree by the round's
    threshold; the carriers (-sign g, h) reproduce the scaled pairs exactly, since |g / p| and h / p round alike.  The refresh
    uses the rows with h != 0, weighted by their instance weight on the weights' grid (absoluteerror_reference.weight_scale)."""

    samples = None

    def update(self):
        if self.samples is None:
            self.samples = []                    # per tree (weighted data): (tree, leaf of every row, its pairs, residuals)
        from absoluteerror_reference import gradient
        from forest_reference import row_stream
        n = len(self.y)
        seed, rnd = int(self.params.get("seed", 0)), self.rounds
        m_grad = self.m.copy()
        resid = (self.y - m_grad).astype(np.float32)
        full = gradient(m_grad, self.y, self.weight)
        u = threshold(rag(full), float(self.params["subsample"]))
        for j in range(self.P):
            gp = sample(full, u, draws(seed, row_stream(rnd, j), n))
            v = self._grow(gp, resid)
            self.m = (self.m + v).astype(np.float32)
            self.weights.append(f32(1))
        self.rounds += 1

    def _grow(self, gp, resid):
        if self.weight is None:
            return super()._grow(gp, resid)
        import absoluteerror_reference as A
        n = len(self.y)
        self.t.y[:] = -np.sign(gp[:, 0]).astype(np.float32)
        self.t.w[:] = gp[:, 1]
        self.t.set_margins(np.zeros(n, np.float32))
        self.t.update()
        model = self.t.model()
        tid = model.num_trees - 1
        leaf = self.O.predict_leaf(model, self.X, tid, tid + 1)[:, 0]
        w_kept = np.where(gp[:, 1] != 0, self.weight, f32(0)).astype(np.float32)
        q = A.refresh(leaf, resid, w_kept, True, A.weight_scale(self.weight, n))
        self.samples.append((tid, leaf, gp, resid))
        vals = {nid: f32(v * self.lr) for nid, v in q.items()}
        self.leaves[tid] = vals
        value = model.tree(tid)["split_cond"].copy()
        for nid, v in vals.items():
            value[nid] = v
        self.rows.append(leaf)
        self.values.append(value)
        return value[leaf]
