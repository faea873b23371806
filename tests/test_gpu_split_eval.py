"""Split evaluation and node expansion on the device (eval_kernel, best_of_blocks, split_is_valid, expand_node through
XGB200BoosterEvalRootSplit) against the NumPy reference of tests/split_reference.py: every reported field bit for bit, on
exact int64 histograms of synthetic quantised rows.  The reference itself is anchored to the oracle by
tests/test_split_reference.py."""
import itertools

import numpy as np
import pytest

import split_reference as R

pytestmark = pytest.mark.gpu
f32 = np.float32
GRID_18 = (1 << 20) + 1          # rows of a matrix trained on the 18-bit grid


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _bits(x):
    return int(f32(x).view(np.uint32))


def _blocks(F):
    """Candidate blocks of the device layout (engine.h feature_layout): full 32-wide groups, then the narrow tail."""
    a, L = F // 32, F % 32
    if a >= 1 and 1 <= L <= 8:
        return [range(32 * g, 32 * g + 32) for g in range(a)] + [range(32 * a, F)]
    return [range(32 * g, min(F, 32 * g + 32)) for g in range(a + (L > 0) or 1)]


def run(xgb, params, hist, tot, cuts, has_missing, n_rows=2, max_g=1.0, max_h=1.0, lower=-np.inf, upper=np.inf, monotone=None,
        feat_mask=None, check_blocks=True):
    """The device's root against the reference; returns the device output."""
    F = len(cuts[0]) - 1
    X = np.zeros((n_rows, F), np.float32)
    if has_missing:
        X[0, 0] = np.nan
    d = xgb.DMatrix(X, label=np.zeros(n_rows, np.float32))
    _be().dmatrix_set_cuts(d.handle, *cuts)
    bp = dict(max_bin=256, **{k: v for k, v in params.items()})
    if monotone is not None:
        bp["monotone_constraints"] = "(" + ",".join(str(int(c)) for c in monotone) + ")"
    bst = xgb.Booster(bp, [d])
    out = _be().eval_root_split(bst.handle, d.handle, hist, tot[0], tot[1], max_g, max_h, lower, upper, feat_mask)
    scales = R.scales_for(max_g, max_h, R.grad_bits_for(n_rows))
    assert out["scales"] == [_bits(s) for s in scales]
    kw = dict(lower=lower, upper=upper, monotone=monotone, feat_mask=feat_mask, colsample_bynode=float(params.get("colsample_bynode", 1.0)),
              seed=int(params.get("seed", 0)))
    ref = R.eval_node(params, hist, cuts[0], cuts[1], cuts[2], has_missing, tot, scales, **kw)
    assert out["root_gain"] == _bits(ref["root_gain"])
    assert out["weight"] == _bits(ref["weight"])

    def same(dev, rb):
        if rb is None:
            assert dev["loss_chg"] == 0 and dev["bin"] == -1
        else:
            assert dev == dict(loss_chg=_bits(rb["loss_chg"]), feature=rb["feature"], bin=rb["bin"], dleft=rb["dleft"], ord=rb["ord"],
                               GL=rb["GL"], HL=rb["HL"]), (dev, rb)

    same(out["best"], ref["best"])
    if check_blocks and kw["colsample_bynode"] >= 1.0:
        blocks = _blocks(F)
        assert len(out["best_group"]) == len(blocks)
        base = np.ones(F, bool) if feat_mask is None else np.asarray(feat_mask, bool)
        for blk, dev in zip(blocks, out["best_group"]):
            m = np.zeros(F, bool); m[list(blk)] = True
            same(dev, R.eval_node(params, hist, cuts[0], cuts[1], cuts[2], has_missing, tot, scales, **dict(kw, feat_mask=base & m))["best"])
    assert out["expanded"] == ref["expanded"]
    for k, v in ref["tree"].items():
        want = [_bits(x) for x in v] if k in ("split_cond", "base_weight", "loss_chg", "sum_hess") else [int(x) for x in v]
        assert out["tree"][k] == want, k
    assert len(out["children"]) == len(ref["children"])
    for dev, rc in zip(out["children"], ref["children"]):
        assert (dev["G"], dev["H"]) == (rc["G"], rc["H"])
        if monotone is not None:
            assert (dev["lower"], dev["upper"]) == (_bits(rc["lower"]), _bits(rc["upper"]))
    return out


LAYOUT_F = [1, 5, 31, 32, 33, 41, 64, 100, 104, 130]


@pytest.mark.parametrize("missing", [0.0, 0.15])
@pytest.mark.parametrize("F", LAYOUT_F)
def test_layouts_bit_exact(xgb, F, missing):
    rng = np.random.default_rng(F * 10 + int(missing > 0))
    for trial, (gmax, hmax) in enumerate([(1 << 21, 1 << 22), (1 << 40, 1 << 41), (3, 2)]):
        nb = rng.choice([1, 2, 8, 33, 255] + ([256] if missing == 0 else []), size=F)
        hist, tot, cuts = R.synth_node(rng, nb, n_rows=int(rng.integers(2, 600)), missing_frac=missing, gmax=gmax, hmax=hmax)
        params = dict(reg_lambda=1.0, min_child_weight=0.0 if trial else 1.0, max_depth=6)
        run(xgb, params, hist, tot, cuts, missing > 0, max_g=f32(rng.uniform(0.5, 50)), max_h=f32(rng.uniform(0.5, 4)))


@pytest.mark.parametrize("F", [5, 33])
def test_layouts_on_the_18_bit_grid(xgb, F):
    rng = np.random.default_rng(180 + F)
    for missing in (0.0, 0.2):
        nb = rng.choice([2, 8, 33, 255], size=F)
        hist, tot, cuts = R.synth_node(rng, nb, n_rows=500, missing_frac=missing, gmax=1 << 18, hmax=1 << 19)
        run(xgb, dict(reg_lambda=1.0, min_child_weight=1.0), hist, tot, cuts, missing > 0, n_rows=GRID_18, max_g=f32(7.5), max_h=f32(1.0))


PARAMS = list(itertools.product([0.0, 1.0, 10.0], [0.0, 0.5], [0.0, 0.7], [0.0, 1.0, 6.5]))


@pytest.mark.parametrize("lam,alpha,mds,mcw", PARAMS)
def test_regularisation_bit_exact(xgb, lam, alpha, mds, mcw):
    rng = np.random.default_rng(int(lam * 100 + alpha * 10 + mds * 1000 + mcw * 7))
    nb = rng.choice([2, 8, 33, 255], size=41)
    hist, tot, cuts = R.synth_node(rng, nb, n_rows=300, missing_frac=0.1, gmax=1 << 21, hmax=1 << 22)
    params = dict(reg_lambda=lam, alpha=alpha, max_delta_step=mds, min_child_weight=mcw)
    run(xgb, params, hist, tot, cuts, True, max_g=f32(40.0), max_h=f32(8.0))


@pytest.mark.parametrize("mds", [0.0, 0.7])
@pytest.mark.parametrize("sign", [1, -1])
def test_monotone_clamping_bit_exact(xgb, sign, mds):
    """Finite node bounds so that the clamp is active; every other feature constrained the other way."""
    rng = np.random.default_rng(11 + sign + int(mds * 10))
    F = 33
    nb = rng.choice([2, 8, 33], size=F)
    hist, tot, cuts = R.synth_node(rng, nb, n_rows=400, missing_frac=0.1, gmax=1 << 21, hmax=1 << 22)
    mono = [sign if f % 2 == 0 else -sign for f in range(F)]
    for lo, hi in [(-np.inf, np.inf), (-0.05, 0.04), (-1e-3, 2e-3)]:
        run(xgb, dict(reg_lambda=1.0, max_delta_step=mds, min_child_weight=0.0), hist, tot, cuts, True, max_g=f32(40.0), max_h=f32(8.0),
            lower=f32(lo), upper=f32(hi), monotone=mono)


@pytest.mark.parametrize("F,src,dst", [(10, 3, 9), (70, 3, 40), (33, 3, 32), (104, 5, 100)])
def test_duplicate_features_the_lower_index_wins(xgb, F, src, dst):
    """Equal candidates in the same block, in different blocks, and in a main block against the tail block."""
    rng = np.random.default_rng(F)
    for trial in range(3):
        nb = rng.choice([2, 4, 8], size=F)
        nb[dst] = nb[src]
        hist, tot, cuts = R.synth_node(rng, nb, n_rows=200, missing_frac=0.1 * trial, gmax=1 << 21, hmax=1 << 22, dup=[(src, dst)])
        # make the duplicated pair the best candidates: scale the rest of the columns' spread down
        for f in range(F):
            if f not in (src, dst):
                hist[f] = 0
                hist[f, 0] = tot
        out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, trial > 0, max_g=f32(8.0), max_h=f32(2.0))
        assert out["best"]["feature"] == src


def _node(bins_gh, missing=(0, 0), extra=()):
    """One feature from explicit (g, h) per bin in grid units (+ missing mass), further features as extra lists."""
    feats = [bins_gh] + list(extra)
    F = len(feats)
    hist = np.zeros((F, 256, 2), np.int64)
    for f, bg in enumerate(feats):
        for b, (g, h) in enumerate(bg):
            hist[f, b] = (g, h)
    tot = (sum(g for g, _ in bins_gh) + missing[0], sum(h for _, h in bins_gh) + missing[1])
    nb = [len(bg) for bg in feats]
    cuts = (np.concatenate([[0], np.cumsum(nb)]).astype(np.int32),
            np.concatenate([f + 0.25 * np.arange(1, k + 1) for f, k in enumerate(nb)]).astype(np.float32), np.arange(F, dtype=np.float32))
    return hist, tot, cuts


U = 1 << 12          # grid units of the hand-made nodes below


def test_scan_order_ties(xgb):
    # equal bins inside one feature (empty bins): the first forward bin wins
    hist, tot, cuts = _node([(-5 * U, 4 * U), (0, 0), (0, 0), (7 * U, 4 * U)])
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, False)
    assert (out["best"]["bin"], out["best"]["dleft"]) == (0, 0)
    # forward against an equal backward candidate (GL = -GR, HL = HR, missing g = 0): the forward one wins
    hist, tot, cuts = _node([(-6 * U, 3 * U), (6 * U, 3 * U)], missing=(0, 2 * U))
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, True)
    assert (out["best"]["bin"], out["best"]["dleft"]) == (0, 0)
    # equal backward candidates (right = the last bin for b = 1, 2, 3): the highest bin wins, i.e. threshold bin 2
    hist, tot, cuts = _node([(5 * U, 3 * U), (0, 0), (0, 0), (-8 * U, 3 * U)], missing=(5 * U, 3 * U))
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, True)
    assert (out["best"]["bin"], out["best"]["dleft"]) == (2, 1)


def test_masked_top_feature_never_wins(xgb):
    rng = np.random.default_rng(5)
    hist, tot, cuts = R.synth_node(rng, [8] * 40, n_rows=300, gmax=1 << 21, hmax=1 << 22)
    first = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, False)
    mask = np.ones(40, np.uint8); mask[first["best"]["feature"]] = 0
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, False, feat_mask=mask)
    assert out["best"]["feature"] != first["best"]["feature"]


def test_min_child_weight_boundary(xgb):
    """HL == min_child_weight is accepted, one grid unit less is not, on each side."""
    unit = float(R.scales_for(1.0, 1.0, 21)[3])
    q = int(6.5 / unit)
    assert q * unit == 6.5
    for side in (0, 1):
        for delta, expand in ((0, True), (-1, False)):
            hq = [q + delta, 3 * q] if side == 0 else [3 * q, q + delta]
            hist, tot, cuts = _node([(-40 << 20, hq[0]), (30 << 20, hq[1])])
            out = run(xgb, dict(reg_lambda=1.0, min_child_weight=6.5), hist, tot, cuts, False)
            assert out["expanded"] == expand, (side, delta)


def test_gamma_and_eps_boundaries(xgb):
    hist, tot, cuts = _node([(-40 << 20, 5 << 22), (30 << 20, 4 << 22)])
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, False)
    loss = np.uint32(out["best"]["loss_chg"]).view(np.float32)
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, gamma=float(loss)), hist, tot, cuts, False)
    assert out["expanded"]
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, gamma=float(np.nextafter(loss, f32(np.inf)))), hist, tot, cuts, False)
    assert not out["expanded"]
    # a best loss_chg in (0, 1e-6] does not expand
    hist, tot, cuts = _node([(-3, 5 << 22), (2, 4 << 22)])
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0), hist, tot, cuts, False)
    loss = np.uint32(out["best"]["loss_chg"]).view(np.float32)
    assert 0 < loss <= 1e-6 and not out["expanded"]


def test_empty_hessian_best_keeps_the_leaf(xgb):
    """The best candidate has HR == 0 (GR != 0): the node stays a leaf although feature 1 has a valid, weaker split."""
    f0 = [(-100 << 10, 5 << 10), (94 << 10, 0)]
    f1 = [(-10 << 10, 2 << 10), (4 << 10, 3 << 10)]
    hist, tot, cuts = _node(f0, extra=[f1])
    params = dict(reg_lambda=0.0, min_child_weight=0.0)
    second = run(xgb, params, hist, tot, cuts, False, feat_mask=np.array([0, 1], np.uint8))
    assert second["expanded"]
    out = run(xgb, params, hist, tot, cuts, False)
    assert out["best"]["feature"] == 0 and not out["expanded"]


def test_all_missing_and_single_bin_features(xgb):
    rng = np.random.default_rng(3)
    for missing in (0.0, 0.3):
        hist, tot, cuts = R.synth_node(rng, [1, 1, 8, 1, 33], n_rows=200, missing_frac=missing, gmax=1 << 21, hmax=1 << 22)
        if missing:
            hist[3] = 0                       # every row of feature 3 is missing
        for mcw in (0.0, 1.0):
            run(xgb, dict(reg_lambda=1.0, min_child_weight=mcw), hist, tot, cuts, missing > 0)


@pytest.mark.parametrize("frac", [0.1, 0.5])
def test_colsample_bynode_at_4096_features(xgb, frac):
    rng = np.random.default_rng(int(frac * 10))
    hist, tot, cuts = R.synth_node(rng, rng.choice([2, 8], size=4096), n_rows=300, missing_frac=0.05, gmax=1 << 21, hmax=1 << 22)
    for seed in (0, 7):
        run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, colsample_bynode=frac, seed=seed), hist, tot, cuts, True)


def test_wide_feature_ids_in_the_split_key(xgb):
    """F = 65 600: the true best sits below 65 536 and a weaker candidate above it; then features 7 and 65 550 tie."""
    F = 65600
    nb = np.full(F, 2)
    cuts = (np.concatenate([[0], np.cumsum(nb)]).astype(np.int32), np.tile(np.array([0.5, 1.5], np.float32), F), np.zeros(F, np.float32))
    tot = (-10 << 20, 8 << 22)
    hist = np.zeros((F, 256, 2), np.int64)
    hist[:, 0] = tot                                        # every feature: all rows in bin 0, no split
    def split(f, g0, h0):
        hist[f, 0] = (g0, h0); hist[f, 1] = (tot[0] - g0, tot[1] - h0)
    split(100, -60 << 20, 4 << 22)
    split(65540, -30 << 20, 4 << 22)
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, max_depth=1), hist, tot, cuts, False, check_blocks=False)
    assert out["best"]["feature"] == 100
    hist[:, 0] = tot; hist[:, 1] = 0
    split(7, -60 << 20, 4 << 22)
    split(65550, -60 << 20, 4 << 22)
    out = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, max_depth=1), hist, tot, cuts, False, check_blocks=False)
    assert out["best"]["feature"] == 7


@pytest.mark.parametrize("F", [33, 100])
def test_depthwise_and_lossguide_expand_the_root_alike(xgb, F):
    rng = np.random.default_rng(F)
    hist, tot, cuts = R.synth_node(rng, rng.choice([2, 8, 33], size=F), n_rows=300, missing_frac=0.1, gmax=1 << 21, hmax=1 << 22)
    mono = [1 if f % 3 == 0 else 0 for f in range(F)]
    for extra in (dict(), dict(max_delta_step=0.7)):
        a = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, max_depth=6, **extra), hist, tot, cuts, True, lower=f32(-0.5), upper=f32(0.5), monotone=mono)
        b = run(xgb, dict(reg_lambda=1.0, min_child_weight=0.0, max_depth=6, grow_policy="lossguide", **extra), hist, tot, cuts, True,
                lower=f32(-0.5), upper=f32(0.5), monotone=mono)
        assert a == b
