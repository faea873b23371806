"""NumPy float64 restatement of the rank:pairwise / rank:ndcg / rank:map gradients (topk pairs) and the ndcg / map metrics, in
the terms of DESIGN.md "Learning to rank".  Used by tests/test_ranking_reference.py (checked against brute force and
scikit-learn) and tests/test_gpu_ranking.py (the device kernels against it)."""
import numpy as np


def group_ptr_from_qid(qid):
    """Runs of equal consecutive qid -> group pointer; qid must not decrease."""
    q = np.asarray(qid)
    if len(q) and np.any(np.diff(q) < 0):
        raise ValueError("qid must be sorted in non-decreasing order")
    starts = np.flatnonzero(np.diff(q)) + 1 if len(q) else np.zeros(0, np.int64)
    return np.concatenate([[0], starts, [len(q)]]).astype(np.int64) if len(q) else np.zeros(1, np.int64)


def order(margin):
    """Stable descending order of the margins, -0.0 read as +0.0, ties in row order."""
    m = np.asarray(margin, np.float64)
    return np.argsort(-np.where(m == 0, 0.0, m), kind="stable")


def gain(y, exp_gain):
    y = np.asarray(y, np.float64)
    return np.exp2(y) - 1.0 if exp_gain else y


def discount(r):
    return 1.0 / np.log2(np.asarray(r, np.float64) + 2.0)


def dcg(y_in_order, exp_gain, k=None):
    y = np.asarray(y_in_order, np.float64)[:k]
    return float(np.sum(gain(y, exp_gain) * discount(np.arange(len(y)))))


def inv_idcg(y, k, exp_gain):
    v = dcg(np.sort(np.asarray(y, np.float64))[::-1], exp_gain, k)
    return 0.0 if v == 0.0 else 1.0 / v


def average_precision(rel_in_order):
    """AP over the whole list: (1/R) sum over the relevant positions r of hits(<= r) / (r + 1); None when R = 0."""
    rel = np.asarray(rel_in_order) > 0
    R = rel.sum()
    if R == 0:
        return None
    hits = np.cumsum(rel)
    return float(np.sum(hits[rel] / (np.flatnonzero(rel) + 1.0)) / R)


def delta_ndcg(y_sorted, a, b, exp_gain, inv):
    """|ΔNDCG| of swapping positions a and b (closed form)."""
    return abs((gain(y_sorted[a], exp_gain) - gain(y_sorted[b], exp_gain)) * (discount(a) - discount(b))) * inv


def map_prefix(y_sorted):
    rel = np.asarray(y_sorted) > 0
    H = np.cumsum(rel).astype(np.float64)
    Q = np.cumsum(np.where(rel, 1.0 / (np.arange(len(rel)) + 1.0), 0.0))
    return H, Q


def delta_map(H, Q, rel_a, a, b):
    """|ΔAP| * R of swapping positions a < b, one of them relevant (closed form from the inclusive prefixes)."""
    ia, ib = 1.0 / (a + 1.0), 1.0 / (b + 1.0)
    if rel_a:
        return abs(H[b] * ib - H[a] * ia - (Q[b] - Q[a]))
    return abs((H[a] + 1.0) * ia - H[b] * ib + (Q[b] - ib - Q[a]))


def _pair_terms(s_sorted, y_sorted, i, j, objective, inv, exp_gain, score_norm):
    """(lambda, h, i is high) of the pairs of margin-order positions (i, j), labels different."""
    if objective == "rank:pairwise":
        delta = np.ones(len(i))
    elif objective == "rank:ndcg":
        delta = delta_ndcg(y_sorted, i, j, exp_gain, inv)
    else:
        H, Q = map_prefix(y_sorted)
        a, b = np.minimum(i, j), np.maximum(i, j)
        ia, ib = 1.0 / (a + 1.0), 1.0 / (b + 1.0)
        rel_a = y_sorted[a] > 0
        d = np.where(rel_a, np.abs(H[b] * ib - H[a] * ia - (Q[b] - Q[a])), np.abs((H[a] + 1.0) * ia - H[b] * ib + (Q[b] - ib - Q[a])))
        delta = d / H[-1]
    i_high = y_sorted[i] > y_sorted[j]
    s_high = np.where(i_high, s_sorted[i], s_sorted[j])
    s_low = np.where(i_high, s_sorted[j], s_sorted[i])
    if score_norm and s_sorted[0] != s_sorted[-1]:
        delta = delta / (np.abs(s_high - s_low) + 0.01)
    sigma = 1.0 / (1.0 + np.exp(-(s_high - s_low)))
    lam = (sigma - 1.0) * delta
    h = np.maximum(sigma * (1.0 - sigma), 1e-16) * delta * 2.0
    return lam, h, i_high


def _group_pairs(s_sorted, y_sorted, objective, k, exp_gain, score_norm):
    """topk: per-position (g, h, |lambda|) sums of one group in margin order, over the pairs (i, j) with i < min(k, n), i < j."""
    n = len(y_sorted)
    acc = np.zeros((3, n))
    kk = min(k, n)
    i = np.repeat(np.arange(kk), n)
    j = np.tile(np.arange(n), kk)
    keep = (j > i) & (y_sorted[i] != y_sorted[j])
    i, j = i[keep], j[keep]
    if len(i) == 0:
        return acc
    lam, h, i_high = _pair_terms(s_sorted, y_sorted, i, j, objective, inv_idcg(y_sorted, kk, exp_gain), exp_gain, score_norm)
    gi = np.where(i_high, lam, -lam)
    for dst, v in ((0, gi), (1, h), (2, -lam)):
        np.add.at(acc[dst], i, v)
    for dst, v in ((0, -gi), (1, h), (2, -lam)):
        np.add.at(acc[dst], j, v)
    return acc


_M64 = (1 << 64) - 1
RANK_PAIR_STREAM = 0x50000000000


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def rng_uniform(seed, stream, idx):
    """csrc/rng.h rng_uniform for one index (Python integers, exact)."""
    h = _splitmix64(_splitmix64(((seed << 32) ^ stream) & _M64) ^ idx)
    return float(np.float32((h >> 40) * (1.0 / 16777216.0)))


def _mean_pairs(rows, y, k, seed, round_, row_offset=0):
    """lambdarank_pair_method=mean: the (document, partner) rows of one group; documents in the stable descending order of their
    labels, each drawing k partners uniformly from the documents outside its label bucket."""
    lab = np.argsort(-y, kind="stable")
    ys = y[lab]
    n = len(y)
    out_i, out_j = [], []
    for q in range(n):
        lo = int(np.searchsorted(-ys, -ys[q], side="left"))
        hi = int(np.searchsorted(-ys, -ys[q], side="right"))
        c = n - (hi - lo)
        if c == 0:
            continue
        for j in range(k):
            u = rng_uniform(seed, RANK_PAIR_STREAM + (round_ << 20) + j, int(rows[lab[q]]) + row_offset)
            t = min(c - 1, int(u * c))
            out_i.append(lab[q])
            out_j.append(lab[t if t < lo else t + (hi - lo)])
    return np.asarray(out_i, np.int64), np.asarray(out_j, np.int64)


def _fix(v):
    """The device's int64 fixed point (2^-32, round half to even) of each pair term."""
    return np.rint(v * 4294967296.0).astype(np.int64)


def gradient(margin, label, group_ptr=None, weight=None, objective="rank:ndcg", k=32, exp_gain=True, normalization=True, score_normalization=True,
             mean=False, seed=0, round_=0):
    """float32 (n, 2) gradient pairs in row order; group_ptr None = one group of all rows; weight one per group.  mean: the
    lambdarank_pair_method=mean pairs of round round_, summed in the device's fixed point."""
    m = np.asarray(margin, np.float32).astype(np.float64)
    y = np.asarray(label, np.float32).astype(np.float64)
    n = len(m)
    ptr = np.array([0, n]) if group_ptr is None else np.asarray(group_ptr, np.int64)
    G = len(ptr) - 1
    wscale = 1.0 if weight is None else G / float(np.sum(np.asarray(weight, np.float32).astype(np.float64)))
    out = np.zeros((n, 2), np.float32)
    for g in range(G):
        b, e = int(ptr[g]), int(ptr[g + 1])
        if e - b < 2:
            continue
        o = order(m[b:e])
        s_sorted, y_sorted = m[b:e][o], y[b:e][o]
        s_sorted = np.where(s_sorted == 0, 0.0, s_sorted)
        if not mean:
            acc = _group_pairs(s_sorted, y_sorted, objective, k, exp_gain, score_normalization)
        else:
            pos = np.empty(e - b, np.int64)
            pos[o] = np.arange(e - b)
            di, dj = _mean_pairs(np.arange(b, e), y[b:e], k, seed, round_)
            fix = np.zeros((3, e - b), np.int64)
            if len(di):
                pi, pj = pos[di], pos[dj]
                lam, h, i_high = _pair_terms(s_sorted, y_sorted, pi, pj, objective, inv_idcg(y_sorted, e - b, exp_gain), exp_gain, score_normalization)
                ph, pl = np.where(i_high, pi, pj), np.where(i_high, pj, pi)
                for dst, at, v in ((0, ph, lam), (0, pl, -lam), (1, pi, h), (1, pj, h), (2, pi, -lam), (2, pj, -lam)):
                    np.add.at(fix[dst], at, _fix(v))
            acc = fix.astype(np.float64) / 4294967296.0
        S = acc[2].sum()
        norm = np.log2(1.0 + S) / S if normalization and S > 0 else 1.0
        scale = norm * (float(np.float32(weight[g])) * wscale if weight is not None else 1.0)
        out[b + o, 0] = (acc[0] * scale).astype(np.float32)
        out[b + o, 1] = (acc[1] * scale).astype(np.float32)
    return out


def metric(margin, label, group_ptr=None, weight=None, name="ndcg", exp_gain=True):
    """ndcg / ndcg@k / ndcg- / ndcg@k- / map / map@k / map- / map@k-: sum w_g v_g / sum w_g."""
    base, minus = (name[:-1], True) if name.endswith("-") else (name, False)
    kind, _, kstr = base.partition("@")
    k = int(kstr) if kstr else None
    m = np.asarray(margin, np.float32).astype(np.float64)
    y = np.asarray(label, np.float32).astype(np.float64)
    ptr = np.array([0, len(m)]) if group_ptr is None else np.asarray(group_ptr, np.int64)
    G = len(ptr) - 1
    w = np.ones(G) if weight is None else np.asarray(weight, np.float32).astype(np.float64)
    vals = np.zeros(G)
    for g in range(G):
        b, e = int(ptr[g]), int(ptr[g + 1])
        ys = y[b:e][order(m[b:e])]
        if kind == "ndcg":
            idcg = dcg(np.sort(ys)[::-1], exp_gain, k)
            vals[g] = (0.0 if minus else 1.0) if idcg == 0.0 else dcg(ys, exp_gain, k) / idcg
        else:
            rel = ys > 0
            R = rel.sum()
            if R == 0:
                vals[g] = 0.0 if minus else 1.0
                continue
            hits = np.cumsum(rel)
            r = np.flatnonzero(rel)
            if k is not None:
                r = r[r < k]
            vals[g] = np.sum(hits[r] / (r + 1.0)) / R
    return float(np.sum(w * vals) / np.sum(w))

