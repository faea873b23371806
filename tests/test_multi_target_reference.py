"""CPU checks of tests/multi_target_reference.py: at T = 1 it is the single-target restatements; on hand-computed cases the
per-target gradients, grids, intercept and metrics are what DESIGN.md "Multi-target regression" says."""
import numpy as np
import pytest

import absoluteerror_reference as AR
import multi_target_reference as MR

f32 = np.float32


def _data(n=257, T=3, seed=0):
    rng = np.random.default_rng(seed)
    Y = rng.normal(0, 1, (n, T)).astype(f32)
    m = rng.normal(0, 1, (n, T)).astype(f32)
    w = rng.uniform(0.1, 2, n).astype(f32)
    return Y, m, w


@pytest.mark.parametrize("objective", MR.OBJECTIVES)
def test_columns_are_single_target_gradients(objective):
    """Target j's pairs are those of a one-column label Y[:, j]: the targets do not see each other."""
    Y, m, w = _data()
    if objective in MR.LOGISTIC:
        Y = (Y > 0).astype(f32)
    if objective == "reg:squaredlogerror":
        Y = np.abs(Y)
    keep = np.random.default_rng(3).uniform(size=len(Y)) < 0.7
    gp = MR.gradient(objective, m, Y, w, scale_pos_weight=2.0, huber_slope=1.5, keep=keep)
    assert gp.shape == (len(Y), 3, 2) and gp.dtype == f32
    for j in range(3):
        one = MR.gradient(objective, m[:, j:j + 1], Y[:, j:j + 1], w, scale_pos_weight=2.0, huber_slope=1.5, keep=keep)
        np.testing.assert_array_equal(gp[:, j], one[:, 0])
    assert np.all(gp[~keep] == 0)


def test_absoluteerror_is_the_single_target_reference():
    Y, m, w = _data()
    gp = MR.gradient("reg:absoluteerror", m, Y, w)
    for j in range(3):
        np.testing.assert_array_equal(gp[:, j], AR.gradient(m[:, j], Y[:, j], w))
    assert MR.intercept("reg:absoluteerror", Y[:, :1], w) == AR.base_score(Y[:, 0], w)


def test_hand_computed_pairs_and_grids():
    Y = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]], f32)
    m = np.array([[0.5, -1.0], [2.0, 0.0], [1.0, 3.0]], f32)
    w = np.array([1.0, 2.0, 0.5], f32)
    gp = MR.gradient("reg:squarederror", m, Y, w, scale_pos_weight=3.0)
    # y == 1 multiplies the row's weight by scale_pos_weight, element by element
    np.testing.assert_array_equal(gp[:, :, 0], np.array([[-1.5, -1.0], [4.0, -6.0], [0.0, 3.0]], f32))
    np.testing.assert_array_equal(gp[:, :, 1], np.array([[3.0, 1.0], [2.0, 6.0], [1.5, 1.5]], f32))
    np.testing.assert_array_equal(MR.target_absmax(gp), np.array([[4.0, 3.0], [6.0, 6.0]], f32))
    ae = MR.gradient("reg:absoluteerror", m, Y, w, scale_pos_weight=3.0)      # no scale_pos_weight outside the RegLossObj family
    np.testing.assert_array_equal(ae[:, :, 0], np.array([[-1.0, -1.0], [2.0, -2.0], [0.0, 0.5]], f32))
    np.testing.assert_array_equal(ae[:, :, 1], np.array([[1.0, 1.0], [2.0, 2.0], [0.5, 0.5]], f32))


def test_pseudohuber_at_zero_and_far():
    Y = np.zeros((2, 1), f32)
    m = np.array([[0.0], [1e3]], f32)
    gp = MR.gradient("reg:pseudohubererror", m, Y)
    assert gp[0, 0, 0] == 0 and gp[0, 0, 1] == 1
    assert abs(gp[1, 0, 0] - 1.0) < 1e-5 and 0 < gp[1, 0, 1] < 1e-8


def test_intercept_is_the_mean_of_the_stumps():
    Y = np.array([[1.0, 10.0], [3.0, 20.0]], f32)
    assert MR.intercept("reg:squarederror", Y) == f32((2.0 + 15.0) / 2)
    w = np.array([3.0, 1.0], f32)
    assert MR.intercept("reg:squarederror", Y, w) == f32((f32(1.5) + f32(12.5)) / 2)
    # the logistic family averages in margin space, then applies the sigmoid once
    P = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 0.0], [1.0, 1.0]], f32)
    b = MR.intercept("binary:logistic", P)
    stumps = [float(f32(-(0.5 * 4 - P[:, j].sum()) / (0.25 * 4))) for j in range(2)]
    assert abs(b - 1 / (1 + np.exp(-np.mean(stumps)))) < 1e-6
    # T = 1 is the stump of the single column
    assert MR.intercept("reg:squarederror", Y[:, 1:]) == f32(15.0)


def test_metrics_over_all_elements():
    Y = np.array([[1.0, 0.0], [0.0, 1.0]], f32)
    P = np.array([[0.5, 0.5], [1.0, 0.0]], f32)
    w = np.array([1.0, 3.0])
    assert MR.metric("rmse", Y, P) == pytest.approx(np.sqrt((0.25 + 0.25 + 1 + 1) / 4))
    assert MR.metric("mae", Y, P, w) == pytest.approx((0.5 + 0.5 + 3 * (1 + 1)) / (2 * 4))
    assert MR.metric("error", Y, P) == pytest.approx((1 + 0 + 1 + 1) / 4)          # only p > 0.5 is class 1
    assert MR.metric("error@0.4", Y, P) == pytest.approx((0 + 1 + 1 + 1) / 4)
    # T = 1: the single-target definition
    y1, p1 = Y[:, :1], P[:, :1]
    assert MR.metric("rmse", y1, p1, w) == pytest.approx(np.sqrt(np.average((p1[:, 0] - y1[:, 0]) ** 2, weights=w)))


def test_shapes():
    s = MR.shapes(10, 3, 5, 12)
    assert s["value"] == (10, 3) and s["pred_leaf"] == (10, 12) and s["pred_contribs"] == (10, 3, 6)
