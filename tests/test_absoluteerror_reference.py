"""CPU checks of the reg:absoluteerror restatement (absoluteerror_reference.py) against the mathematics: upstream's unweighted
Quantile is numpy's "weibull" quantile, the fixed-point weighted rule agrees with upstream's float-CDF WeightedQuantile except
where that CDF lands within rounding of alpha * total, a refreshed leaf minimises the leaf's weighted absolute error, and the
oracle's carrier pairs are the absolute-error pairs."""
import numpy as np
import pytest

import absoluteerror_reference as A

f32 = np.float32


def _adversarial(rng):
    yield np.array([3.5], f32)
    yield np.array([2.0, -1.0], f32)
    yield np.full(7, 1.25, f32)
    yield np.array([0.0, -0.0, 0.0, -0.0], f32)
    yield np.array([-0.0, 1.0, -2.0, 0.0, 0.0], f32)
    yield np.array([1e-45, -1e-45, 3e38, -3e38, 0.0], f32)
    yield np.round(rng.standard_normal(1001) * 4).astype(f32)          # many ties
    yield rng.standard_normal(200000).astype(f32)


@pytest.mark.parametrize("alpha", [0.5, 0.1, 0.9, 0.0, 1.0])
def test_quantile_is_weibull(alpha):
    rng = np.random.default_rng(1)
    sets = list(_adversarial(rng)) + [rng.standard_normal(n).astype(f32) * 10 for n in (3, 4, 5, 10, 11, 12345)]
    for v in sets:
        q = A.quantile(v, alpha)
        ref = np.quantile(v.astype(np.float64), alpha, method="weibull")
        assert np.isfinite(q) or not np.isfinite(ref)
        assert abs(float(q) - ref) <= 1e-6 * max(1.0, abs(ref)), (len(v), alpha, q, ref)


def test_zero_sign_does_not_matter():
    a = A.quantile(np.array([-0.0, -0.0, 1.0], f32))
    assert np.signbit(a) == np.False_ and a == 0
    v = np.array([-0.0, 0.0, 2.0, -0.0], f32)
    assert A.keys(v)[0] == A.keys(v)[1]
    assert A.segmented_quantile(v)[0].view(np.uint32) == A.segmented_quantile(v[::-1])[0].view(np.uint32)


def _boundary_gap(v, w, alpha):
    """|exact cumulative weight at upstream's pick boundary - alpha * total| relative to the total."""
    s, order = A._sorted(v)
    cum = np.cumsum(np.asarray(w, np.float64)[order])
    t = alpha * cum[-1]
    return np.min(np.abs(cum - t)) / cum[-1]


def test_weighted_agrees_with_float_cdf_except_at_boundary():
    rng = np.random.default_rng(2)
    differ = 0
    for trial in range(300):
        n = int(rng.integers(1, 400))
        v = np.round(rng.standard_normal(n) * 3, 1).astype(f32)
        # weights on the fixed-point grid of their maximum, so the integer rule sees them exactly
        w = (rng.integers(1, 1 << 20, n) * 2.0 ** -20).astype(f32)
        sh = A.weight_scale(w, n)
        hq = A.h_q(w, sh)
        assert np.array_equal(hq.astype(np.float64) / float(sh), w.astype(np.float64))
        a, b = A.weighted_quantile_hq(v, hq), A.upstream_weighted_quantile(v, w)
        if a != b:
            differ += 1
            assert _boundary_gap(v, w, 0.5) <= 4 * n * 2.0 ** -24, (trial, a, b)
    assert differ < 10


def test_constructed_case_where_float_cdf_differs():
    """Second half of the weights a copy of the first, so the exact cumulative weight meets total / 2 at the middle: the
    integer rule picks the last value of the first half, while upstream's float CDF falls short of its rounded threshold."""
    for seed in range(200):
        rng = np.random.default_rng(seed)
        half = (rng.integers(1 << 18, 1 << 20, 64) * 2.0 ** -20).astype(f32)
        w = np.concatenate([half, half[::-1]])
        v = np.arange(len(w), dtype=f32)
        hq = A.h_q(w, A.weight_scale(w, len(w)))
        assert 2 * int(hq[:64].sum()) == int(hq.sum())
        a, b = A.weighted_quantile_hq(v, hq), A.upstream_weighted_quantile(v, w)
        assert a == 63.0
        if b != a:
            assert b == 64.0
            return
    pytest.fail("no seed separates the two rules")


@pytest.mark.parametrize("weighted", [False, True])
def test_refresh_minimises_absolute_error(weighted):
    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 8, 51, 500):
        r = np.round(rng.standard_normal(n) * 5, 2).astype(f32)
        w = rng.integers(1, 50, n).astype(f32) if weighted else np.ones(n, f32)
        leaf = np.zeros(n, np.int64)
        sh = A.weight_scale(w, n)
        q = A.refresh(leaf, r, w, weighted, sh)[0]
        loss = lambda c: float(np.sum(w.astype(np.float64) * np.abs(r.astype(np.float64) - c)))
        best = min(loss(c) for c in r.astype(np.float64))
        assert loss(float(q)) <= best * (1 + 1e-12) + 1e-9, (n, q)


def test_segmented_quantile_segments_and_exclusions():
    rng = np.random.default_rng(4)
    n, S = 5000, 37
    v = rng.standard_normal(n).astype(f32)
    seg = rng.integers(-1, S - 3, n)                  # the last segments stay empty
    out = A.segmented_quantile(v, seg, None, S)
    for s in range(S):
        rows = v[seg == s]
        if len(rows) == 0:
            assert np.isnan(out[s])
        else:
            assert out[s] == A.quantile(rows)
    w = rng.integers(0, 4, n).astype(f32)
    out_w = A.segmented_quantile(v, seg, w, S)
    hq = A.h_q(w, A.weight_scale(w, n))
    for s in range(S):
        m = (seg == s) & (w != 0)
        assert (np.isnan(out_w[s]) and not m.any()) or out_w[s] == A.weighted_quantile_hq(v[m], hq[m])


def test_trainer_carriers_and_loss():
    rng = np.random.default_rng(5)
    n, F = 3000, 6
    X = rng.standard_normal((n, F)).astype(f32)
    y = (X[:, 0] * 2 + rng.laplace(size=n)).astype(f32)
    w = rng.integers(1, 4, n).astype(f32)
    t = A.AbsErrorTrainer(dict(objective="reg:absoluteerror", max_depth=4, eta=0.5), X, y, weight=w)
    assert t.base_score == A.base_score(y, w)
    losses = []
    for _ in range(5):
        m0 = t.m.copy()
        t.update()
        gp = t.t.gpair()[:, 0, :]
        np.testing.assert_array_equal(gp, A.gradient(m0, y, w))
        losses.append(float(np.sum(w * np.abs(y - t.m))))
    assert losses[-1] < losses[0]
    from oracle import gbt_oracle as O
    np.testing.assert_array_equal(O.predict_margin(t.model(), X)[:, 0], t.m)


def test_nan_orders_above_inf():
    v = np.array([np.nan, 1.0, np.inf, -np.nan, -np.inf], f32)
    k = A.keys(v)
    assert k[0] == k[3] and k[0] > k[2] > k[1] > k[4]
    assert int(k.max()) < 0xFFFFFFFF


@pytest.mark.parametrize("extra", [dict(num_parallel_tree=3, subsample=0.6, seed=5), dict(booster="dart", rate_drop=0.3, one_drop=1, seed=7)])
def test_trainer_forest_and_dart_bookkeeping(extra):
    """The margins the restatement advances equal the model it returns, evaluated from scratch: a forest's trees at weight 1 in
    model order, a dart model's trees at their final weights."""
    from oracle import gbt_oracle as O
    import dart_reference as DR
    rng = np.random.default_rng(6)
    n, F = 3000, 6
    X = rng.standard_normal((n, F)).astype(f32)
    y = (X[:, 0] * 2 + rng.laplace(size=n)).astype(f32)
    t = A.AbsErrorTrainer(dict(objective="reg:absoluteerror", max_depth=4, eta=0.5, **extra), X, y)
    for _ in range(4):
        t.update()
    model = t.model()
    P = int(extra.get("num_parallel_tree", 1))
    assert model.num_trees == 4 * P and len(t.weights) == 4 * P
    if "booster" in extra:
        assert any(w != 1 for w in t.weights)
        np.testing.assert_allclose(DR.predict_margin(model, X, t.weights)[:, 0], t.m, rtol=0, atol=1e-5)
    else:
        np.testing.assert_array_equal(O.predict_margin(model, X)[:, 0], t.m)
        for tid, vals in t.leaves.items():          # the refresh scaled by fl(eta / P)
            off = int(model["tree_offset"][tid])
            assert all(model["split_cond"][off + nid] == v for nid, v in vals.items())
