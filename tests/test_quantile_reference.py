"""tests/quantile_reference.py checked on its own (no GPU): parameter parsing, the gradient pairs and their carriers, the
per-target refresh at the ends of [0, 1], the base score and the quantile metric."""
import numpy as np
import pytest

import absoluteerror_reference as A
import quantile_reference as QR

f32 = np.float32


@pytest.mark.parametrize("value, want", [
    ("0.5", [0.5]), (0.25, [0.25]), ("(0.1,0.5,0.9)", [0.1, 0.5, 0.9]), ("[0.1, 0.5, 0.9]", [0.1, 0.5, 0.9]),
    ([0.1, 0.9], [0.1, 0.9]), ((0.0, 1.0), [0.0, 1.0]), (np.array([0.2, 0.4]), [0.2, 0.4]), (np.float64(0.3), [0.3]),
    (" [ 0.05 ,0.95 ] ", [0.05, 0.95]),
])
def test_parse_accepts(value, want):
    np.testing.assert_array_equal(QR.parse_alpha(value), np.array(want, np.float32))


@pytest.mark.parametrize("value", ["", "()", "[]", "1.5", "-0.1", "(0.1,2)", "abc", "0.1;0.2", "nan"])
def test_parse_rejects(value):
    with pytest.raises(QR.QuantileAlphaError):
        QR.parse_alpha(value)


def test_gradient_pairs_and_carriers():
    rng = np.random.default_rng(1)
    n, alpha = 1000, QR.parse_alpha("(0.1,0.5,0.9)")
    y = rng.standard_normal(n).astype(f32)
    m = rng.standard_normal((n, 3)).astype(f32)
    m[:10, 1] = y[:10]                                           # d == 0 counts as d >= 0
    w = rng.uniform(0, 3, n).astype(f32)
    gp = QR.gradient(m, y, alpha, w)
    for j, a in enumerate(alpha):
        d = (m[:, j] - y).astype(f32)
        g = np.where(d >= 0, f32(f32(1) - a) * w, f32(-a) * w).astype(f32)
        np.testing.assert_array_equal(gp[:, j, 0], g)
        np.testing.assert_array_equal(gp[:, j, 1], w)
        c = QR.carriers(m[:, j], y, a)
        np.testing.assert_array_equal(((f32(0) - c) * w).astype(f32), g)     # squared error at margin 0 on the carriers
    keep = rng.random(n) < 0.5
    gk = QR.gradient(m, y, alpha, w, keep)
    assert np.all(gk[~keep] == 0) and np.array_equal(gk[keep], gp[keep])


@pytest.mark.parametrize("weighted", [False, True])
def test_refresh_ends_are_min_and_max(weighted):
    rng = np.random.default_rng(2)
    n = 5000
    leaf = rng.integers(0, 9, n)
    resid = rng.standard_normal(n).astype(f32)
    h = rng.uniform(0.5, 2, n).astype(f32) if weighted else np.ones(n, f32)
    h[rng.random(n) < 0.1] = 0                                   # rows outside the sample take no part
    sh = A.weight_scale(h, n)
    lo = QR.refresh(leaf, resid, h, weighted, sh, 0.0)
    hi = QR.refresh(leaf, resid, h, weighted, sh, 1.0)
    for nid in lo:
        rows = (leaf == nid) & (h != 0)
        assert lo[nid] == resid[rows].min() and hi[nid] == resid[rows].max()


def test_refresh_at_alpha_minimises_the_pinball_loss():
    rng = np.random.default_rng(3)
    v = rng.standard_normal(2001).astype(f32)
    for a in (0.1, 0.3, 0.9):
        q = QR.refresh(np.zeros(len(v), np.int64), v, np.ones(len(v), f32), False, 1.0, a)[0]
        grid = np.linspace(-3, 3, 601).astype(f32)
        loss = [QR.pinball(v, np.full(len(v), c, f32), [a]) for c in grid]
        assert QR.pinball(v, np.full(len(v), q, f32), [a]) <= min(loss) + 1e-6


def test_metric_matches_direct_formula():
    rng = np.random.default_rng(4)
    n, alpha = 777, np.array([0.05, 0.5, 0.95], f32)
    y = rng.standard_normal(n).astype(f32)
    p = rng.standard_normal((n, 3)).astype(f32)
    w = rng.uniform(0, 2, n).astype(f32)
    direct = 0.0
    for i in range(n):
        for j in range(3):
            d = float(y[i]) - float(p[i, j])
            direct += float(w[i]) * (float(alpha[j]) * d if d >= 0 else (float(alpha[j]) - 1.0) * d)
    direct /= 3 * float(np.sum(w, dtype=np.float64))
    assert abs(QR.pinball(y, p, alpha, w) - direct) <= 1e-6 * abs(direct)
    assert QR.pinball(y, p[:, :1], alpha[:1]) == pytest.approx(np.mean(np.maximum(alpha[0] * (y - p[:, 0]), (alpha[0] - 1) * (y - p[:, 0]))), rel=1e-6)


@pytest.mark.parametrize("weighted", [False, True])
def test_base_score_is_mean_of_quantiles(weighted):
    rng = np.random.default_rng(5)
    y = rng.standard_normal(10001).astype(f32)
    w = rng.uniform(0, 3, len(y)).astype(f32) if weighted else None
    alpha = np.array([0.1, 0.5, 0.9], f32)
    qs = [A.segmented_quantile(y, None, w, 1, float(a))[0] for a in alpha]
    sw = len(y) if w is None else float(np.cumsum(w.astype(np.float64))[-1])
    assert QR.base_score(y, alpha, w) == f32((float(qs[0]) + float(qs[1]) + float(qs[2])) / 3 * sw / (sw + 1e-6))
    # one alpha of 0.5: the absolute-error base score, scaled by sw / (sw + 1e-6)
    assert QR.base_score(y, [0.5], w) == f32(float(A.base_score(y, w)) * sw / (sw + 1e-6))
    scale = len(y) / (len(y) + 1e-6)
    assert QR.base_score(y, [0.0]) == f32(float(y.min()) * scale) and QR.base_score(y, [1.0]) == f32(float(y.max()) * scale)
