"""What travels with the row ids through the partition (run with `pytest -m gpu` on an H100).

Constant-hessian objectives carry g alone and the deeper histograms add the constant h_q of h == 1; the line-aligned row
copy of 3 full groups + an 8-wide tail (F = 101 ... 104) holds the tail bytes in the pad of each row's 128 B line, so the
gathered levels stop gathering them from bins_tail.  Both must leave every result bit-identical.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from util import assert_same_structure, first_structural_difference, max_leaf_diff, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODE_TRAINING_TAIL = 4      # build_histogram_ex: the tail source of the training path
MODE_G_ONLY_PAYLOAD = 8     # build_histogram_ex: g by position, h == 1.0f for every row


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _subset(xgb, n, F, frac, ordered, seed=23):
    X, y = synth(n, F, seed, "reg")
    rng = np.random.default_rng(5)
    gpair = np.stack([rng.standard_normal(n).astype(np.float32) * 3, rng.random(n).astype(np.float32) + 0.01], axis=1)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster({"max_bin": 256}, [d])
    m = max(1, int(n * frac))
    rows = np.random.default_rng(9).choice(n, size=m, replace=False).astype(np.uint32)
    if ordered:
        rows.sort()
    return d, b, rows, gpair[:m]


# F = 100: aligned copy, 4-wide tail by position; F = 104: 8-wide tail in the aligned line; F = 36: one group, tail by
# position; F = 130: two group chunks
@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("n,F,frac", [(120000, 100, 0.25), (50000, 104, 0.3), (70001, 36, 0.4), (20000, 130, 0.5)])
def test_g_only_payload_gather_bit_exact(xgb, oracle, n, F, frac, ordered):
    """The gathered levels' G-only-payload variant: g by position, the H plane gets rint(1.0f * sh) per row whatever h the
    caller holds, which is exactly what the (g,h) path computes when h == 1."""
    d, b, rows, gp_pos = _subset(xgb, n, F, frac, ordered)
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gp_pos, mode=MODE_TRAINING_TAIL | MODE_G_ONLY_PAYLOAD, row_ids=rows)
    assert kernel == "hist_gather_kernel"
    gq = np.zeros(n, np.int32); hq = np.zeros(n, np.int32)
    gq[rows] = np.rint(gp_pos[:, 0] * scales[0]).astype(np.int32)
    hq[rows] = np.int32(np.rint(np.float32(1.0) * scales[1]))
    bins = _be().dmatrix_get_bins(d.handle, 256)
    np.testing.assert_array_equal(hist, oracle.build_hist_fixed(bins, gq, hq, rows=rows))


@pytest.mark.parametrize("ordered", [True, False])
def test_eight_wide_tail_from_the_aligned_line_bit_exact(xgb, oracle, ordered):
    """F = 104: the 8 tail bytes come from the pad of the row's aligned line, (g,h) by position."""
    n, F = 50000, 104
    d, b, rows, gp_pos = _subset(xgb, n, F, 0.3, ordered)
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gp_pos, mode=MODE_TRAINING_TAIL, row_ids=rows)
    assert kernel == "hist_gather_kernel"
    gq = np.zeros(n, np.int32); hq = np.zeros(n, np.int32)
    gq[rows] = np.rint(gp_pos[:, 0] * scales[0]).astype(np.int32)
    hq[rows] = np.rint(gp_pos[:, 1] * scales[1]).astype(np.int32)
    bins = _be().dmatrix_get_bins(d.handle, 256)
    np.testing.assert_array_equal(hist, oracle.build_hist_fixed(bins, gq, hq, rows=rows))


_TRAIN = r"""
import json, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import sagemaker_xgboost_container_b200 as xgb
from util import synth
X, y = synth(200000, 100, 41, "reg", quantised=False)
d = xgb.DMatrix(X, label=y)
bst = xgb.train(json.loads(sys.argv[2]), d, num_boost_round=4, verbose_eval=False)
be = xgb.get_backend()
m = be.booster_export_model(bst.handle)
out = {k: np.asarray(v) for k, v in m.items()}
out["cached_margin"] = be.booster_cached_margin(bst.handle, d.handle, 1)
np.savez(sys.argv[3], **out)
"""


def _train_in_subprocess(tmp_path, params, no_consth):
    env = dict(os.environ)
    env.pop("B200XGB_NO_CONSTH", None)
    if no_consth:
        env["B200XGB_NO_CONSTH"] = "1"          # read once per process: the two models are trained in two processes
    out = str(tmp_path / ("model_%d.npz" % no_consth))
    r = subprocess.run([sys.executable, "-s", "-c", _TRAIN, ROOT, json.dumps(params), out], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return dict(np.load(out))


@pytest.mark.parametrize("extra", [dict(max_depth=6), dict(grow_policy="lossguide", max_leaves=24, max_depth=6)])
def test_constant_hessian_path_is_bit_identical(tmp_path, extra):
    """reg:squarederror on 100 features: the model trained with the constant-hessian path (G-only root pass, g-only partition
    payload, constant h_q in the deeper histograms) equals the one trained with B200XGB_NO_CONSTH=1 in every bit."""
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, eta=0.3, **extra)
    fast = _train_in_subprocess(tmp_path, params, False)
    plain = _train_in_subprocess(tmp_path, params, True)
    assert (fast["left"] != -1).sum() > 4 * 8, "the trees should really split"
    assert fast.keys() == plain.keys()
    for k in fast:
        np.testing.assert_array_equal(fast[k], plain[k], err_msg=k)


@pytest.mark.parametrize("F", [100, 104])
def test_missing_values_in_the_tail_block_match_the_oracle(xgb, oracle, F):
    """Missing values everywhere, the tail features included (bin 255 in the tail bytes: by position for F = 100, in the
    aligned line for F = 104)."""
    n, rounds = 60000, 5
    X, y = synth(n, F, 57, "reg", quantised=False, missing_frac=0.08)
    assert np.isnan(X[:, 96:]).any()
    y = (y + 0.8 * np.nan_to_num(X[:, 98]) - 0.6 * np.nan_to_num(X[:, 99], nan=1.0)).astype(np.float32)      # make the tail features matter
    params = dict(objective="reg:squarederror", tree_method="hist", max_bin=256, max_depth=6, eta=0.3)
    d = xgb.DMatrix(X, label=y)
    bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    m = _be().booster_export_model(bst.handle)
    mr = oracle.train(params, X, y, rounds).model()
    assert first_structural_difference(m, mr) is None, "tree structure differs first at tree %s" % first_structural_difference(m, mr)
    assert_same_structure(m, mr)
    assert max_leaf_diff(m, mr) <= 1e-5
    assert np.isin(np.arange(96, F), m["split_index"][m["left"] != -1]).any(), "a tail feature should be split on"
