"""The survival restatement in tests/survival_reference.py against the mathematics, independently of recall: AFT gradients
against numerical derivatives of a scipy.stats likelihood, Cox against the Breslow partial likelihood, the metrics against
closed forms.  No GPU needed."""
import numpy as np
import pytest
from scipy import stats

import survival_reference as SR

SCIPY = {"normal": stats.norm, "logistic": stats.logistic, "extreme": stats.gumbel_l}


def _intervals(rng, n, kind):
    t = np.exp(rng.normal(1.0, 0.6, n))
    if kind == "uncensored":
        return t, t.copy()
    if kind == "right":
        return t, np.full(n, np.inf)
    if kind == "left":
        return np.zeros(n), t
    return t, t * rng.uniform(1.2, 3.0, n)


def _nll(dist, lo, hi, m, s):
    D = SCIPY[dist]
    if np.all(lo == hi):
        z = (np.log(lo) - m) / s
        return -(D.logpdf(z) - np.log(s * lo))
    fu = np.where(np.isinf(hi), 1.0, D.cdf((np.log(np.where(np.isinf(hi), 1.0, hi)) - m) / s))
    fl = np.where(lo <= 0, 0.0, D.cdf((np.log(np.where(lo <= 0, 1.0, lo)) - m) / s))
    return -np.log(fu - fl)


@pytest.mark.parametrize("dist", sorted(SR.DISTS))
@pytest.mark.parametrize("kind", ["uncensored", "right", "left", "interval"])
@pytest.mark.parametrize("sigma", [0.7, 1.0, 2.0])
def test_aft_gradient_is_the_derivative_of_the_likelihood(dist, kind, sigma):
    rng = np.random.default_rng(hash((dist, kind, sigma)) % 2**32)
    n = 200
    lo, hi = _intervals(rng, n, kind)
    lo, hi = lo.astype(np.float32).astype(np.float64), hi.astype(np.float32).astype(np.float64)
    s = float(np.float32(sigma))
    m = (np.log(np.where(lo > 0, lo, hi)) + rng.uniform(-1.0, 1.0, n)).astype(np.float32).astype(np.float64)
    g, h = SR.aft_grad_hess(dist, lo, hi, m, sigma)
    eps = 1e-4
    num_g = (_nll(dist, lo, hi, m + eps, s) - _nll(dist, lo, hi, m - eps, s)) / (2 * eps)
    num_h = (_nll(dist, lo, hi, m + eps, s) - 2 * _nll(dist, lo, hi, m, s) + _nll(dist, lo, hi, m - eps, s)) / eps**2
    inside = (np.abs(num_g) < 15) & (num_h < 15) & (num_h > 1e-6)
    assert inside.mean() > 0.8
    np.testing.assert_allclose(g[inside], num_g[inside], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(h[inside], num_h[inside], rtol=2e-3, atol=1e-5)


@pytest.mark.parametrize("dist", sorted(SR.DISTS))
@pytest.mark.parametrize("kind", ["uncensored", "right", "left", "interval"])
def test_aft_gradient_is_finite_and_clipped_at_extreme_margins(dist, kind):
    rng = np.random.default_rng(3)
    lo, hi = _intervals(rng, 64, kind)
    for mval in (-40.0, 40.0):
        for sigma in (0.7, 1.0, 2.0):
            gp = SR.aft_gradient(np.full(64, mval, np.float32), lo, hi, None, dist, sigma)
            assert np.all(np.isfinite(gp))
            assert np.all((gp[:, 0] >= -15) & (gp[:, 0] <= 15))
            assert np.all((gp[:, 1] >= np.float32(1e-16)) & (gp[:, 1] <= 15))


def _breslow_nll(m, y):
    """Negative Breslow partial log-likelihood: -sum over events of (m_i - ln sum_{|y_j| >= |y_i|} exp(m_j))."""
    a = np.abs(y)
    out = 0.0
    for i in np.nonzero(y > 0)[0]:
        out -= m[i] - np.log(np.sum(np.exp(m[a >= a[i]])))
    return out


def test_cox_gradient_is_the_derivative_of_the_partial_likelihood_without_ties():
    rng = np.random.default_rng(11)
    n = 60
    t = rng.permutation(n).astype(np.float64) + 1.0
    y = np.where(rng.random(n) < 0.7, t, -t).astype(np.float32)
    m = rng.normal(0, 0.5, n).astype(np.float32).astype(np.float64)
    gp = SR.cox_gradient(m, y)
    eps = 1e-5
    for i in range(n):
        e = np.zeros(n); e[i] = eps
        fg = (_breslow_nll(m + e, y) - _breslow_nll(m - e, y)) / (2 * eps)
        fh = (_breslow_nll(m + e, y) - 2 * _breslow_nll(m, y) + _breslow_nll(m - e, y)) / eps**2
        assert abs(gp[i, 0] - fg) <= 1e-5 * max(1.0, abs(fg))
        assert abs(gp[i, 1] - fh) <= 2e-3 * max(1.0, abs(fh))


def _cox_vectorised(m, y, w):
    """Breslow with upstream's tie rule, written independently: D from each tie-group head, R and S over the events so far."""
    a = np.abs(y)
    order = np.argsort(a, kind="stable")
    e = np.exp(m[order].astype(np.float64))
    suf = np.cumsum(e[::-1])[::-1]
    D = suf[np.searchsorted(a[order], a[order], side="left")]
    ev = (y[order] > 0).astype(np.float64)
    R, S = np.cumsum(ev / D), np.cumsum(ev / D**2)
    g, h = np.empty(len(m)), np.empty(len(m))
    g[order] = (e * R - ev) * w[order]
    h[order] = (e * R - e * e * S) * w[order]
    return g, h


def test_cox_gradient_with_ties_and_weights_matches_the_tie_rule():
    rng = np.random.default_rng(12)
    n = 3000
    t = rng.integers(1, 200, n).astype(np.float32)
    y = np.where(rng.random(n) < 0.6, t, -t).astype(np.float32)
    m = rng.normal(0, 1, n).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    gp = SR.cox_gradient(m, y, w)
    g, h = _cox_vectorised(m, y, w)
    np.testing.assert_allclose(gp[:, 0], g, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(gp[:, 1], h, rtol=1e-5, atol=1e-6)


def test_cox_tie_rule_differs_from_the_exact_derivative():
    """Two events tied at t = 1: upstream's R of the first counts only itself, the exact Breslow derivative counts both."""
    y = np.array([1.0, 1.0, 2.0, -3.0], np.float32)
    m = np.array([0.1, -0.2, 0.3, 0.0], np.float64)
    gp = SR.cox_gradient(m, y)
    eps = 1e-6
    e = np.zeros(4); e[1] = eps
    exact = (_breslow_nll(m + e, y) - _breslow_nll(m - e, y)) / (2 * eps)
    e0 = np.zeros(4); e0[0] = eps
    exact0 = (_breslow_nll(m + e0, y) - _breslow_nll(m - e0, y)) / (2 * eps)
    assert abs(gp[1, 0] - exact) < 1e-5                 # the last event of the group sees both
    assert abs(gp[0, 0] - exact0) > 1e-2                # the first one does not


def test_metrics_against_closed_forms():
    rng = np.random.default_rng(5)
    n = 500
    lo, hi = _intervals(rng, n, "interval")
    lo[:100] = hi[:100]
    hi[100:200] = np.inf
    lo[200:300] = 0.0
    m = rng.normal(1.0, 1.0, n).astype(np.float32)
    w = rng.uniform(0.5, 2, n).astype(np.float32)
    lo32, hi32 = lo.astype(np.float32), hi.astype(np.float32)
    L, H, M, W = lo32.astype(np.float64), hi32.astype(np.float64), m.astype(np.float64), w.astype(np.float64)
    z = (np.log(L[:100]) - M[:100])
    want = np.concatenate([-(stats.norm.logpdf(z) - np.log(L[:100])),
                           -np.log(np.where(np.isinf(H[100:]), 1.0, stats.norm.cdf(np.log(np.where(np.isinf(H[100:]), 1, H[100:])) - M[100:]))
                                   - np.where(L[100:] <= 0, 0.0, stats.norm.cdf(np.log(np.where(L[100:] <= 0, 1, L[100:])) - M[100:])))])
    assert SR.aft_nloglik(m, lo32, hi32, w) == pytest.approx(np.sum(want * W) / W.sum(), rel=1e-10)
    p = np.exp(M)
    assert SR.interval_accuracy(m, lo32, hi32, w) == pytest.approx(np.sum(((p >= L) & (p <= H)) * W) / W.sum(), rel=1e-12)
    y = np.where(rng.random(n) < 0.5, 1, -1) * rng.integers(1, 50, n).astype(np.float32)
    assert SR.cox_nloglik(m, y) == pytest.approx(_breslow_nll(M, y) / np.sum(y > 0), rel=1e-10)


def test_carrier_gives_back_the_pairs():
    rng = np.random.default_rng(2)
    gp = np.stack([rng.normal(0, 3, 10000), rng.uniform(1e-16, 15, 10000)], axis=1).astype(np.float32)
    gp[:10] = 0.0
    y, w = SR.carrier(gp)
    g = (np.float32(0) - y) * w
    np.testing.assert_array_equal(np.float32(1) * w, gp[:, 1])
    ulps = np.abs(g.view(np.int32).astype(np.int64) - gp[:, 0].view(np.int32).astype(np.int64))
    assert ulps.max() <= 1 and (ulps == 0).mean() > 0.85


def test_aft_parameters_reach_the_engine():
    from sagemaker_xgboost_container_b200 import core
    assert core._check_unapplied("aft_loss_distribution", "logistic") == "logistic"
    assert core._check_unapplied("aft_loss_distribution_scale", "1.5") == "1.5"
