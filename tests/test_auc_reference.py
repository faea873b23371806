"""tests/auc_reference.py pinned down on the CPU: the one-vs-rest ROC against scikit-learn, binary PR-AUC against numerical
integration of an independently built precision(recall) curve, closed forms, and the combination over ranks."""
import math

import numpy as np
import pytest
from scipy import integrate
from sklearn.metrics import roc_auc_score

import auc_reference as AR


def _softmax32(m):
    m = np.asarray(m, np.float32)
    e = np.exp(m - m.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)


def _tied_probs(rng, n, K, levels=4):
    """Probabilities with heavy ties: every row's margins come from a few levels."""
    return _softmax32(rng.integers(0, levels, (n, K)).astype(np.float32) * 0.7)


@pytest.mark.parametrize("K", [3, 10])
@pytest.mark.parametrize("weighted", [False, True])
def test_multiclass_roc_matches_sklearn_ovr_weighted(K, weighted):
    rng = np.random.default_rng(K + 10 * weighted)
    n = 3000
    p = _tied_probs(rng, n, K)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    got = AR.multiclass_auc(p, y, w)
    sw = None if w is None else w.astype(np.float64)           # scikit-learn sums float32 weights in float32
    want = roc_auc_score(y.astype(int), p.astype(np.float64), multi_class="ovr", average="weighted", sample_weight=sw, labels=list(range(K)))
    assert got == pytest.approx(want, rel=1e-12, abs=1e-14)


@pytest.mark.parametrize("weighted", [False, True])
def test_binary_roc_matches_sklearn(weighted):
    rng = np.random.default_rng(3 + weighted)
    n = 5000
    s = np.round(rng.standard_normal(n), 1).astype(np.float32)
    y = (rng.random(n) < 0.3).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    wd = AR._weights(n, w)
    tp, fp = AR.curve(s, wd * y, wd * (1.0 - y))
    got = AR.roc_area(tp, fp) / (tp[-1] * fp[-1])
    assert got == pytest.approx(roc_auc_score(y, s, sample_weight=None if w is None else w.astype(np.float64)), rel=1e-12)


def _pr_by_quadrature(s, y, w):
    """Integrate precision over recall with scipy, segment by segment, from an independent walk of the tie blocks."""
    s = np.asarray(s, np.float32).astype(np.float64)
    w = np.ones(len(s)) if w is None else np.asarray(w, np.float32).astype(np.float64)
    y = np.asarray(y, np.float64)
    levels = np.unique(s)[::-1]
    pts = [(0.0, 0.0)]
    for v in levels:
        sel = s >= v
        pts.append((float(np.sum(w[sel] * y[sel])), float(np.sum(w[sel] * (1 - y[sel])))))
    P = pts[-1][0]
    total = 0.0
    for (tp0, fp0), (tp1, fp1) in zip(pts[:-1], pts[1:]):
        if tp1 == tp0:
            continue

        def precision(r, tp0=tp0, fp0=fp0, tp1=tp1, fp1=fp1):
            tp = r * P
            fp = fp0 + (fp1 - fp0) * (tp - tp0) / (tp1 - tp0)
            return tp / (tp + fp)

        val, _ = integrate.quad(precision, tp0 / P, tp1 / P, epsabs=1e-14, epsrel=1e-13, limit=200)
        total += val
    return total


@pytest.mark.parametrize("seed", range(6))
def test_binary_pr_matches_quadrature(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(20, 400))
    s = np.round(rng.standard_normal(n), 1).astype(np.float32)
    y = (rng.random(n) < rng.uniform(0.1, 0.9)).astype(np.float32)
    if seed % 3 == 2:                      # soft labels: fractional positive shares
        y = np.round(rng.random(n), 2).astype(np.float32)
    y[0], y[1] = 1.0, 0.0
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if seed % 2 else None
    got = AR.aucpr(s, y, w)
    assert got == pytest.approx(_pr_by_quadrature(s, y, w), rel=1e-9)


def test_closed_forms():
    # a perfect ranking
    s = np.array([4, 3, 2, 1, 0], np.float32)
    y = np.array([1, 1, 0, 0, 0], np.float32)
    assert AR.aucpr(s, y) == 1.0
    p = np.eye(3, dtype=np.float32)[[0, 1, 2, 0]] * 0.8 + 0.2 / 3
    assert AR.multiclass_auc(p, [0, 1, 2, 0]) == 1.0
    assert AR.multiclass_aucpr(p, [0, 1, 2, 0]) == 1.0
    # all scores tied: P / (P + N)
    y = np.array([1, 0, 0, 1, 0, 0, 0], np.float32)
    assert AR.aucpr(np.zeros(7, np.float32), y) == pytest.approx(2 / 7, rel=1e-15)
    w = np.array([1, 2, 3, 4, 5, 6, 7], np.float32)
    assert AR.aucpr(np.zeros(7, np.float32), y, w) == pytest.approx(5 / 28, rel=1e-15)
    # one negative above P tied positives: the integral of r P / (r P + 1) over [0, 1] = 1 - ln(1 + P) / P
    for P in (1, 2, 7, 1000):
        s = np.array([1.0] + [0.5] * P, np.float32)
        y = np.array([0.0] + [1.0] * P, np.float32)
        assert AR.aucpr(s, y) == pytest.approx(1.0 - math.log(1.0 + P) / P, rel=1e-13)


def test_negative_zero_ties_with_positive_zero():
    s = np.array([1.0, 0.0, -0.0, -1.0], np.float32)
    y = np.array([1, 0, 1, 0], np.float32)
    tp, fp = AR.curve(s, y, 1 - y)
    assert len(tp) == 3
    s2 = np.array([1.0, -0.0, 0.0, -1.0], np.float32)
    assert AR.aucpr(s, y) == AR.aucpr(s2, y)


def test_degenerate_and_invalid():
    # an absent class: nan, no error
    p = _softmax32(np.random.default_rng(0).standard_normal((50, 3)))
    y = np.array([0, 1] * 25, np.float32)
    assert math.isnan(AR.multiclass_auc(p, y))
    assert math.isnan(AR.multiclass_aucpr(p, y))
    # binary: one class only raises, labels outside [0, 1] raise
    with pytest.raises(ValueError, match="only contains pos or neg"):
        AR.aucpr(np.arange(5, dtype=np.float32), np.ones(5, np.float32))
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        AR.aucpr(np.arange(3, dtype=np.float32), np.array([0, 1, 2], np.float32))
    assert math.isnan(AR.binary_aucpr(np.arange(5, dtype=np.float32), np.zeros(5, np.float32)))


def test_ranks():
    rng = np.random.default_rng(7)
    p = _tied_probs(rng, 400, 3)
    y = rng.integers(0, 3, 400).astype(np.float32)
    w = rng.uniform(0.5, 2.0, 400).astype(np.float32)
    # one rank is the single-rank value; the ROC sum rule over ranks is not the mean of per-rank values
    assert AR.ranks_multiclass_auc([(p, y, w)]) == AR.multiclass_auc(p, y, w)
    two = AR.ranks_multiclass_auc([(p[:200], y[:200], w[:200]), (p[200:], y[200:], w[200:])])
    per = [(AR.class_pieces(p[a:b], y[a:b], w[a:b])) for a, b in ((0, 200), (200, 400))]
    want = (sum((per[0][c][0] + per[1][c][0]) / (per[0][c][2] * per[0][c][3] + per[1][c][2] * per[1][c][3]) * (per[0][c][2] + per[1][c][2]) for c in range(3))
            / sum(per[0][c][2] + per[1][c][2] for c in range(3)))
    assert two == pytest.approx(want, rel=1e-15)
    # aucpr: the mean of the ranks' values; a rank without positives makes it nan; binary raises on global totals only
    s = rng.standard_normal(400).astype(np.float32)
    yb = (rng.random(400) < 0.4).astype(np.float32)
    v0, v1 = AR.binary_aucpr(s[:200], yb[:200]), AR.binary_aucpr(s[200:], yb[200:])
    assert AR.ranks_aucpr([v0, v1]) == (v0 + v1) / 2
    yb2 = yb.copy()
    yb2[200:] = 0.0
    vals = [AR.binary_aucpr(s[:200], yb2[:200]), AR.binary_aucpr(s[200:], yb2[200:])]
    tot = [AR.binary_pieces(s[:200], yb2[:200])[1:], AR.binary_pieces(s[200:], yb2[200:])[1:]]
    assert math.isnan(AR.ranks_aucpr(vals, tot))
    with pytest.raises(ValueError, match="only contains pos or neg"):
        AR.ranks_aucpr([math.nan, math.nan], [(0.0, 5.0), (0.0, 7.0)])
