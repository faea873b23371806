"""Exact restatement of the quantile cuts and the binning that the product (csrc/quantile.cu, misc.cu bin_kernel) and the
oracle (oracle/gbt_oracle.c cuts_from_distinct, orc_bin) share, and of the multi-GPU cut recipe (booster.cu ensure_binned:
capped per-rank summaries merged in rank order).  Written from the definition, not from either implementation.

- Distinct values: NaN and the matrix's `missing` value are missing; +inf and -inf are values; -0.0 and +0.0 are one value,
  represented by +0.0.
- Weights: every finite float32 is an integer multiple of 2^-149, so each distinct value's weight is summed exactly as an
  integer (int64 when it provably cannot overflow, else Python integers).  The sums are then converted to double, and the
  conversion is asserted exact: that assertion is the *exact regime*, inside which every correct implementation that sums
  the weights in double, in whatever order, gets these cuts bit for bit.  Since every partial sum of the weights is an integer
  multiple of the smallest weight unit and no larger than the total, the regime is simply "total weight < 2^53 units".
- Cuts: nb = min(max_bin, 256), or 255 when the matrix has a missing value.  With m <= nb distinct values the cuts are the
  distinct values after the first; otherwise cut k (k = 1 .. nb-1) is the distinct value after the first one whose inclusive
  cumulative weight reaches W k / nb in the definition's double arithmetic, kept when larger than the previous cut.  Both add
  the end cut last + (|last| + 1e-5f), in float32 (+inf at FLT_MAX); the min is first - (|first| + 1e-5f).  An all-missing
  feature gets the one cut 1e-5f and the min -1e-5f.
- Bins: searchsorted(cuts, v, side="right") clipped to the last bin; missing -> 255.
"""
import numpy as np

EPS = np.float32(1e-5)
MISSING_BIN = 255
RANK_CAP = 2048          # points per feature of a rank's summary (csrc/misc.h kRankSummaryCap)
EXACT_BITS = 53


class NotExact(AssertionError):
    """The weights leave the exact regime: a double sum of them may round."""


def _missing_mask(col, missing):
    m = np.isnan(col)
    if missing is not None and not np.isnan(missing):
        m |= col == np.float32(missing)
    return m


def _weight_units(w):
    """float32 weights -> (int array k, e) with w == k * 2^e exactly, e as large as possible.  k is int64 when every sum
    of them fits, else an object array of Python integers."""
    w = np.ascontiguousarray(w, np.float32)
    if not np.all(np.isfinite(w)) or np.any(w < 0):
        raise ValueError("weights must be finite and >= 0")
    bits = w.view(np.uint32).astype(np.int64)
    ef = (bits >> 23) & 0xFF
    mant = np.where(ef == 0, bits & 0x7FFFFF, (bits & 0x7FFFFF) | 0x800000)
    shift = np.maximum(ef, 1) - 1                      # w == mant * 2^(shift - 149)
    nz = mant != 0
    if not nz.any():
        return np.zeros(len(w), np.int64), 0
    ctz = np.zeros_like(mant)
    t = mant.copy()
    for b in (16, 8, 4, 2, 1):                         # trailing zero bits of the nonzero mantissas
        low = nz & ((t & ((1 << b) - 1)) == 0)
        ctz += np.where(low, b, 0)
        t = np.where(low, t >> b, t)
    base = int((shift + ctz)[nz].min())                # the smallest unit every weight is a multiple of
    up = shift - base
    if int(up.max()) + 24 + int(len(w)).bit_length() < 62:
        k = np.where(up >= 0, mant << np.maximum(up, 0), mant >> np.maximum(-up, 0))
        return k.astype(np.int64), base - 149
    k = np.array([int(a) << int(u) if u >= 0 else int(a) >> int(-u) for a, u in zip(mant.tolist(), up.tolist())], dtype=object)
    return k, base - 149


def _to_double(units, e):
    """exact integer sums (units of 2^e, >= 0) -> float64, asserting the conversion is exact.  The bound is on the
    integer itself, not on its significant bits: below 2^53 units every partial sum in any order is exact too."""
    if len(units) and max(int(u) for u in (units.tolist() if units.dtype == object else [units.max()])) >= (1 << EXACT_BITS):
        raise NotExact("a weight sum reaches 2^53 units of the smallest weight: double sums of it may round")
    out = np.array([float(int(u)) for u in units.tolist()], np.float64) if units.dtype == object else units.astype(np.float64)
    return np.ldexp(out, e)


def in_exact_regime(weights, n=None):
    """True when every partial sum of `weights` (None: n unit weights) is exact in double"""
    if weights is None:
        return n < (1 << EXACT_BITS)
    k, _ = _weight_units(weights)
    return int(k.sum()) < (1 << EXACT_BITS)


def distinct(col, units, missing=np.nan):
    """sorted distinct values of one column (float32, zero as +0.0) and their exact weight sums (integer units)"""
    col = np.asarray(col, np.float32)
    keep = ~_missing_mask(col, missing)
    v = col[keep]
    v = np.where(v == 0, np.float32(0), v).astype(np.float32)
    d, inv = np.unique(v, return_inverse=True)
    u = units[keep]
    if u.dtype == object:
        cw = np.array([0] * len(d), dtype=object)
        for i, x in zip(inv.tolist(), u.tolist()):
            cw[i] += x
    else:
        cw = np.zeros(len(d), np.int64)
        np.add.at(cw, inv, u)
    return d, cw


def _cumsum(cw):
    if cw.dtype == object:
        out, acc = [], 0
        for x in cw.tolist():
            acc += x
            out.append(acc)
        return np.array(out, dtype=object)
    return np.cumsum(cw)


def end_cut(last):
    with np.errstate(over="ignore"):
        return np.float32(last) + (np.abs(np.float32(last)) + EPS)


def min_value(first):
    with np.errstate(over="ignore"):
        return np.float32(first) - (np.abs(np.float32(first)) + EPS)


def cuts_from_distinct(d, cw, e, nb):
    """the shared cut rule on distinct values d (sorted float32) with exact weights cw (integer units of 2^e)"""
    m = len(d)
    if m == 0:
        return np.array([EPS], np.float32)
    if m <= nb:
        cuts = list(d[1:])
    else:
        # cum + cw[i] in the definition's loop is the inclusive running sum, exact in double inside the regime: the loop
        # stops at the first i whose running sum is not below the target
        C = _to_double(_cumsum(cw), e)
        _to_double(cw, e)
        W = float(C[-1])
        cuts, last = [], d[0]
        for k in range(1, nb):
            target = W * float(k) / float(nb)
            i = int(np.searchsorted(C, target, side="left"))
            j = min(i + 1, m - 1)
            if d[j] > last:
                cuts.append(d[j])
                last = d[j]
    cuts.append(end_cut(d[-1]))
    return np.array(cuts, np.float32)


def _assemble(per_feature, nb_mins):
    ptrs = np.zeros(len(per_feature) + 1, np.int32)
    for f, c in enumerate(per_feature):
        ptrs[f + 1] = ptrs[f] + len(c)
    vals = np.concatenate(per_feature).astype(np.float32) if per_feature else np.zeros(0, np.float32)
    return ptrs, vals, np.array(nb_mins, np.float32)


def has_missing_values(X, missing=np.nan):
    return bool(_missing_mask(np.asarray(X, np.float32), missing).any())


def num_bins(max_bin, has_missing):
    nb = min(int(max_bin), 256)
    return min(nb, 255) if has_missing else nb


def make_cuts(X, max_bin=256, weights=None, missing=np.nan):
    """(ptrs int32 [F+1], vals float32, mins float32 [F], has_missing) of the single-GPU cuts"""
    X = np.asarray(X, np.float32)
    n, F = X.shape
    units, e = _weight_units(np.ones(n, np.float32) if weights is None else weights)
    hm = has_missing_values(X, missing)
    nb = num_bins(max_bin, hm)
    per, mins = [], []
    for f in range(F):
        d, cw = distinct(X[:, f], units, missing)
        per.append(cuts_from_distinct(d, cw, e, nb))
        mins.append(min_value(d[0]) if len(d) else -EPS)
    return _assemble(per, mins) + (hm,)


def bin_matrix(X, ptrs, vals, missing=np.nan):
    """uint8 [n][F]: upper bound of each value among its feature's cuts, clipped to the last bin; missing -> 255"""
    X = np.asarray(X, np.float32)
    n, F = X.shape
    out = np.empty((n, F), np.uint8)
    for f in range(F):
        c = vals[ptrs[f]:ptrs[f + 1]]
        col = X[:, f]
        b = np.minimum(np.searchsorted(c, col, side="right"), len(c) - 1)
        b[_missing_mask(col, missing)] = MISSING_BIN
        out[:, f] = b
    return out


def rank_summary(d, cw, e, cap=RANK_CAP):
    """one rank's summary of one feature: (values, exact weights in units of 2^e).  Exact when m <= cap; else point k
    (k = 0 .. cap-1) is the first distinct value whose cumulative weight reaches W (k+1) / cap (the last value at the
    latest), after the first distinct value; repeated points collapse, and a point's weight is the difference of the
    cumulative weights."""
    m = len(d)
    if m <= cap:
        return d, cw
    Ci = _cumsum(cw)
    C = _to_double(Ci, e)
    W = float(C[-1])
    idx = [0]
    for k in range(cap):
        target = W * float(k + 1) / float(cap)
        i = int(np.searchsorted(C[:m - 1], target, side="left"))
        if d[i] > d[idx[-1]]:
            idx.append(i)
    vals = d[idx]
    ws = [Ci[idx[0]]] + [Ci[idx[j]] - Ci[idx[j - 1]] for j in range(1, len(idx))]
    return vals, np.array(ws, dtype=object if Ci.dtype == object else np.int64)


def merge(summaries):
    """summaries of the ranks in rank order -> one (values, weights): stable sort by value, equal values add weights"""
    vs = np.concatenate([s[0] for s in summaries]).astype(np.float32)
    ws = np.concatenate([np.asarray(s[1], dtype=object) for s in summaries])
    order = np.argsort(vs, kind="stable")
    out_v, out_w = [], []
    for i in order.tolist():
        if out_v and out_v[-1] == vs[i]:
            out_w[-1] += ws[i]
        else:
            out_v.append(vs[i])
            out_w.append(ws[i])
    return np.array(out_v, np.float32), np.array(out_w, dtype=object)


def rank_cuts(X, max_bin, row_bounds, weights=None, missing=np.nan, cap=RANK_CAP):
    """(ptrs, vals, mins) of the multi-GPU recipe with rows [row_bounds[r], row_bounds[r+1]) as rank r's shard"""
    X = np.asarray(X, np.float32)
    n, F = X.shape
    units, e = _weight_units(np.ones(n, np.float32) if weights is None else weights)
    nb = num_bins(max_bin, has_missing_values(X, missing))
    per, mins = [], []
    for f in range(F):
        sums = []
        for r in range(len(row_bounds) - 1):
            b, en = int(row_bounds[r]), int(row_bounds[r + 1])
            d, cw = distinct(X[b:en, f], units[b:en], missing)
            sums.append(rank_summary(d, cw, e, cap))
        d, cw = merge(sums)
        per.append(cuts_from_distinct(d, cw, e, nb))
        mins.append(min_value(d[0]) if len(d) else -EPS)
    return _assemble(per, mins)
