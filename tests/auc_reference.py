"""Double-precision restatement of the AUC family (DESIGN.md "AUC family"): binary aucpr, one-vs-rest multi-class auc and
aucpr, and their combination over ranks.  The scores are what the engine reads (the sigmoid / margin of a one-output model,
predict()'s softmax probabilities of a multi-class one); -0.0 counts as +0.0.  Rows are walked from the highest score to
the lowest in blocks of tied scores; row i adds w_i y_i to the positives and w_i (1 - y_i) to the negatives.

The functions return the unnormalised pieces the engine all-reduces, and the metric values built from them:
- `curve(s, pos, neg)`: the (tp, fp) running sums at the end of every tie block;
- `roc_area`, `pr_area`: the area terms of one class (ROC unnormalised, PR in recall units);
- `binary_aucpr`, `multiclass_auc`, `multiclass_aucpr`: one rank's value (nan for a class without positive or negative weight);
- `ranks_aucpr`, `ranks_multiclass_auc`: the value over several ranks.
"""
import math

import numpy as np

AUC_ERROR = "Check failed: !auc_error AUC: the dataset only contains pos or neg samples"


def _scores(s):
    s = np.asarray(s, dtype=np.float32).astype(np.float64)
    return np.where(s == 0.0, 0.0, s)


def curve(s, pos, neg):
    """(tp, fp) at the end of each block of tied scores, walked from the highest score down."""
    s = _scores(s)
    order = np.argsort(-s, kind="stable")
    ss = s[order]
    tp = np.cumsum(np.asarray(pos, np.float64)[order])
    fp = np.cumsum(np.asarray(neg, np.float64)[order])
    if len(ss) == 0:
        return tp, fp
    ends = np.flatnonzero(np.append(ss[1:] != ss[:-1], True))
    return tp[ends], fp[ends]


def roc_area(tp, fp):
    """The tie-aware trapezoids: sum over blocks of (fp1 - fp0) (tp1 + tp0) / 2 (binary auc = this / (P N))."""
    area = 0.0
    tp0 = fp0 = 0.0
    for t, f in zip(tp.tolist(), fp.tolist()):
        area += (f - fp0) * (t + tp0) * 0.5
        tp0, fp0 = t, f
    return area


def pr_segment(tp0, fp0, tp1, fp1, P):
    """Davis-Goadrich: fp linear in tp between the two block ends; the area under precision = r / (a r + b), r = tp / P."""
    if tp1 == tp0:
        return 0.0
    h = (fp1 - fp0) / (tp1 - tp0)
    a = 1.0 + h
    b = (fp0 - h * tp0) / P
    r0, r1 = tp0 / P, tp1 / P
    if b != 0.0:    # the log difference ln(a r1 + b) - ln(a r0 + b), evaluated as log1p (DESIGN.md "AUC family")
        return ((r1 - r0) - b / a * math.log1p(a * (r1 - r0) / (a * r0 + b))) / a
    return (r1 - r0) / a


def pr_area(tp, fp):
    """Binary aucpr of one class: the segments from (0, 0) through every block end, P = the last tp."""
    if len(tp) == 0 or tp[-1] <= 0.0:
        return 0.0
    P = float(tp[-1])
    area = 0.0
    tp0 = fp0 = 0.0
    for t, f in zip(tp.tolist(), fp.tolist()):
        area += pr_segment(tp0, fp0, t, f, P)
        tp0, fp0 = t, f
    return area


def _weights(n, w):
    return np.ones(n) if w is None else np.asarray(w, np.float32).astype(np.float64)


def binary_pieces(s, y, w=None):
    """(aucpr area, P, N) of a one-output model's scores; labels are the positive share and must lie in [0, 1]."""
    y = np.asarray(y, np.float32).astype(np.float64)
    if np.any(~((y >= 0.0) & (y <= 1.0))):
        raise ValueError("label must be in [0, 1] for aucpr")
    w = _weights(len(y), w)
    tp, fp = curve(s, w * y, w * (1.0 - y))
    P = float(tp[-1]) if len(tp) else 0.0
    N = float(fp[-1]) if len(fp) else 0.0
    return pr_area(tp, fp), P, N


def binary_aucpr(s, y, w=None):
    """One rank's binary aucpr: nan when the rank has no positive or no negative weight."""
    area, P, N = binary_pieces(s, y, w)
    return area if P > 0.0 and N > 0.0 else math.nan


def class_pieces(prob, y, w=None):
    """Per class c of an (n, K) probability matrix: (roc area, pr area, P_c, N_c), positives (int)label == c."""
    prob = np.asarray(prob, np.float32)
    n, K = prob.shape
    lab = np.asarray(y, np.float32).astype(np.int64)
    w = _weights(n, w)
    out = []
    for c in range(K):
        yc = (lab == c).astype(np.float64)
        tp, fp = curve(prob[:, c], w * yc, w * (1.0 - yc))
        P = float(tp[-1]) if len(tp) else 0.0
        N = float(fp[-1]) if len(fp) else 0.0
        out.append((roc_area(tp, fp), pr_area(tp, fp), P, N))
    return out


def multiclass_auc(prob, y, w=None, pieces=None):
    """sum_c auc_c P_c / sum_c P_c over one rank; nan when a class has no positive or no negative weight."""
    return ranks_multiclass_auc([(prob, y, w)], None if pieces is None else [pieces])


def multiclass_aucpr(prob, y, w=None, pieces=None):
    """The unweighted mean over classes of each class's aucpr; nan when a class has no positive or no negative weight."""
    pieces = class_pieces(prob, y, w) if pieces is None else pieces
    total = 0.0
    for _, pr, P, N in pieces:
        total += pr if P > 0.0 and N > 0.0 else math.nan
    return total / len(pieces)


def ranks_multiclass_auc(shards, per=None):
    """Several ranks, shards = [(prob, y, w), ...]: per class the sums over ranks of the area, of P_c N_c and of P_c
    (per: the ranks' class_pieces, when already computed)."""
    per = [class_pieces(*sh) for sh in shards] if per is None else per
    K = len(per[0])
    area = [sum(p[c][0] for p in per) for c in range(K)]
    pn = [sum(p[c][2] * p[c][3] for p in per) for c in range(K)]
    pc = [sum(p[c][2] for p in per) for c in range(K)]
    num = den = 0.0
    for c in range(K):
        if pn[c] == 0.0:
            return math.nan
        num += area[c] / pn[c] * pc[c]
        den += pc[c]
    return num / den


def ranks_aucpr(values, totals=None):
    """aucpr over ranks: the mean of each rank's value.  totals = [(P, N), ...] of a binary model: the error of binary auc
    when the global totals have no positive or no negative weight."""
    if totals is not None:
        P = sum(t[0] for t in totals)
        N = sum(t[1] for t in totals)
        if not (P > 0.0 and N > 0.0):
            raise ValueError(AUC_ERROR)
    return sum(values) / len(values)


def aucpr(s, y, w=None):
    """Binary aucpr on one rank, raising like the engine when there is no positive or no negative weight."""
    area, P, N = binary_pieces(s, y, w)
    if not (P > 0.0 and N > 0.0):
        raise ValueError(AUC_ERROR)
    return area
