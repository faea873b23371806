"""The restatement of sampling_method=gradient_based (tests/gradient_sampling_reference.py) against its definition: the threshold
solves sum min(1, rag / u) = k, agrees with an O(n^2) solve and with upstream's float sort-and-scan rule, and the edge cases
(ties, zero pairs, k = 0, k >= n, non-finite and denormal rag) have their documented results.  CPU only."""
import numpy as np
import pytest

import gradient_sampling_reference as G

f32 = np.float32


def _rag(rng, n, kind):
    if kind == "normal":
        g, h = rng.standard_normal(n), rng.uniform(0.0, 1.0, n)
    elif kind == "ties":
        g, h = np.round(rng.standard_normal(n), 1), np.ones(n)
    elif kind == "zeros":
        g, h = rng.standard_normal(n), rng.uniform(0.0, 1.0, n)
        z = rng.random(n) < 0.3
        g[z], h[z] = 0.0, 0.0
    else:                                        # "wide": magnitudes over many binades
        g, h = rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n)), rng.uniform(0.0, 1.0, n)
    return G.rag(np.stack([g, h], 1).astype(f32))


@pytest.mark.parametrize("kind", ["normal", "ties", "zeros", "wide"])
@pytest.mark.parametrize("subsample", [0.01, 0.2, 0.5, 0.99])
def test_threshold_solves_the_kept_sum(kind, subsample):
    r = _rag(np.random.default_rng(1), 20000, kind)
    u = G.threshold(r, subsample)
    k = G.target(len(r), subsample)
    if k >= np.count_nonzero(r):
        assert u == 0
        return
    np.testing.assert_allclose(G.kept_sum(r, u), k, rtol=1e-6)


@pytest.mark.parametrize("kind", ["normal", "ties", "zeros"])
@pytest.mark.parametrize("subsample", [0.01, 0.5, 0.99])
def test_threshold_matches_brute_force_and_upstream(kind, subsample):
    rng = np.random.default_rng(2)
    for n in (7, 50, 300):
        r = _rag(rng, n, kind)
        k = G.target(n, subsample)
        u = G.threshold(r, subsample)
        brute = G.brute_threshold(r, k)
        if brute is None:                        # k >= the rows with rag > 0: every row kept
            assert u == 0 and k >= int(np.count_nonzero(r))
            continue
        np.testing.assert_allclose(float(u), brute, rtol=1e-6)
        up = G.upstream_threshold(r, subsample)
        if up is not None:                       # upstream's float scan rounds once per row
            np.testing.assert_allclose(float(up), brute, rtol=max(1e-6, n * 2.0 ** -24))
            np.testing.assert_allclose(float(u), float(up), rtol=max(1e-6, n * 2.0 ** -23))


def test_k_zero_takes_one_row():
    r = _rag(np.random.default_rng(3), 50, "normal")
    assert int(f32(50) * f32(0.01)) == 0
    assert G.target(50, 0.01) == 1
    u = G.threshold(r, 0.01)
    np.testing.assert_allclose(G.kept_sum(r, u), 1.0, rtol=1e-6)
    assert G.upstream_threshold(r, 0.01) is None         # upstream's rule has no valid index there


@pytest.mark.parametrize("subsample", [0.999, 0.6])
def test_k_at_least_the_nonzero_rows_keeps_everything(subsample):
    gp = np.zeros((1000, 2), f32)
    gp[:500] = np.random.default_rng(4).standard_normal((500, 2)).astype(f32) ** 2 + f32(0.1)
    # k = 999 (or 600) >= 500 rows with rag > 0
    u, out = G.gradient_based_sample(gp, subsample, seed=5)
    assert u == 0
    assert np.array_equal(out.view(np.uint32), gp.view(np.uint32))


def test_all_zero_pairs():
    gp = np.zeros((100, 2), f32)
    u, out = G.gradient_based_sample(gp, 0.3)
    assert u == 0 and not np.any(out)


def test_ties_only():
    gp = np.tile(np.array([[0.5, 1.0]], f32), (1000, 1))
    r = G.rag(gp)
    u = G.threshold(r, 0.25)
    # every row has p = r / u = 0.25 (to rounding): u = 4 r
    np.testing.assert_allclose(float(u), 4.0 * float(r[0]), rtol=1e-6)
    _, out = G.gradient_based_sample(gp, 0.25, seed=1)
    kept = out[:, 1] != 0
    np.testing.assert_allclose(out[kept], gp[kept] * 4.0, rtol=1e-6)


def test_non_finite_rag_kept_unscaled_and_left_out_of_the_sums():
    rng = np.random.default_rng(6)
    gp = rng.standard_normal((2000, 2)).astype(f32) ** 2
    gp[:5, 0] = np.inf
    gp[5:8, 0] = np.nan
    r = G.rag(gp)
    u = G.threshold(r, 0.3)
    k = G.target(2000, 0.3)
    fin = np.isfinite(r)
    np.testing.assert_allclose(G.kept_sum(r[fin], u) + 8, k, rtol=1e-6)
    _, out = G.gradient_based_sample(gp, 0.3, seed=2)
    assert np.array_equal(out[:8].view(np.uint32), gp[:8].view(np.uint32))


def test_denormal_rag():
    gp = np.zeros((400, 2), f32)
    gp[:, 0] = np.arange(1, 401, dtype=np.uint32).view(f32)        # denormal g, h = 0: rag = |g|... flushed by g * g to 0
    gp[200:, 0] = f32(1e-25)                                          # g * g underflows: rag 0 although g != 0
    gp[300:, 1] = f32(2e-19)                                          # lambda h^2 is denormal
    r = G.rag(gp)
    assert np.all(r[:300] == 0) and np.all(r[300:] > 0)
    u, out = G.gradient_based_sample(gp, 0.5, seed=3)
    # 100 rows with rag > 0 and k = 200: every row kept as it is (rag == 0 rows included: u == 0)
    assert u == 0 and np.array_equal(out.view(np.uint32), gp.view(np.uint32))
    u, out = G.gradient_based_sample(gp, 0.1, seed=3)                 # k = 40 of the 100
    np.testing.assert_allclose(G.kept_sum(r, u), 40, rtol=1e-6)
    assert not np.any(out[:300])                                      # p = 0: dropped


def test_threshold_with_one_huge_row():
    r = np.concatenate([np.full(999, 1e-3, f32), [f32(3e38)]])
    u = G.threshold(r, 0.1)
    # the huge row is kept with p = 1; the other 999 share k - 1 = 99
    np.testing.assert_allclose(float(u), 999e-3 / 99, rtol=1e-5)


def test_sample_rule():
    gp = np.array([[1.0, 1.0], [0.0, 0.0], [4.0, 0.0], [-0.25, 0.5]], f32)
    u = f32(2.0)
    d = np.array([0.9, 0.0, 0.0, 0.1], f32)
    out = G.sample(gp, u, d)
    r = G.rag(gp)
    p0 = r[0] / u
    assert np.array_equal(out[0], [0, 0]) if d[0] >= p0 else True
    assert np.array_equal(out[1], [0, 0])                             # zero pair stays zero
    assert np.array_equal(out[2], gp[2])                              # p >= 1: unscaled
    p3 = r[3] / u
    assert d[3] < p3
    assert out[3, 0] == gp[3, 0] / p3 and out[3, 1] == gp[3, 1] / p3


def test_statistics_of_the_sample():
    rng = np.random.default_rng(8)
    n = 200000
    gp = np.stack([rng.standard_normal(n), rng.uniform(0.01, 1.0, n)], 1).astype(f32)
    u, out = G.gradient_based_sample(gp, 0.2, seed=9)
    p = np.minimum(1.0, G.rag(gp).astype(np.float64) / float(u))
    kept = out[:, 1] != 0
    k = G.target(n, 0.2)
    sd = np.sqrt(np.sum(p * (1 - p)))
    assert abs(kept.sum() - k) <= 5 * sd
    g = gp[:, 0].astype(np.float64)
    sd_g = np.sqrt(np.sum(g * g * (1 - p) / p))
    assert abs(out[:, 0].astype(np.float64).sum() - g.sum()) <= 5 * sd_g
    assert np.all(kept[p >= 1]) and np.array_equal(out[p >= 1], gp[p >= 1])
