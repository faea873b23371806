"""The gathered histogram passes end every (CTA, node) segment with plain stores of the CTA's accumulators into a partial slot
of its own, and one reduce launch adds the partial slots of each built node to its pool slot (run with `pytest -m gpu` on an
H100).  The sums are exact integers, so the histograms must equal the oracle's int64 mirror bit for bit, and every model
must equal the one trained with the previous RED.ADD.64 flush (B200XGB_HIST_RED_FLUSH=1) bit for bit.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_exact_growth import grow_and_compare
from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODE_FORCE_GATHER = 1       # build_histogram_ex: the contiguous pass through hist_gather_kernel
MODE_TRAINING_TAIL = 4      # build_histogram_ex: the tail source of the training path
ROWS_PER_CTA = 4096         # hist.cu kMinRowsPerCta: a launch splits T rows over ceil(T / 4096) CTAs, at most one per SM
WINDOW = 8064               # rows between two overflow checks on the 18-bit grid (matrices above 2^20 rows)


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


@pytest.fixture(scope="module")
def skewed(xgb):
    """2.4 M x 100 where most rows share one bin per feature and one large gradient: the accumulators of that bin cross the
    spill threshold every window, and the final flush of a segment holds up to a window's worth of the largest g_q in one
    entry (the tail replicas' sum of such an entry does not fit 32 bits and must still come out exact)."""
    n, F = 2_400_000, 100
    rng = np.random.default_rng(61)
    X = np.zeros((n, F), np.float32)
    rare = rng.random((n, F)) < 0.03
    X[rare] = np.round(rng.standard_normal(rare.sum()) * 32).astype(np.float32) / 32
    y = rng.standard_normal(n).astype(np.float32)
    gpair = np.empty((n, 2), np.float32)
    gpair[:, 0] = np.where(rng.random(n) < 0.9, np.float32(4.0), rng.standard_normal(n).astype(np.float32))
    gpair[:, 1] = np.where(rng.random(n) < 0.9, np.float32(2.0), rng.random(n).astype(np.float32))
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster({"max_bin": 256}, [d])
    return d, b, gpair


def _check(d, gp, hist, scales, oracle, rows):
    n = _be().dmatrix_num_row(d.handle)
    gq = np.zeros(n, np.int32); hq = np.zeros(n, np.int32)
    idx = np.arange(n) if rows is None else rows
    gq[idx] = np.rint(gp[:, 0] * scales[0]).astype(np.int32)
    hq[idx] = np.rint(gp[:, 1] * scales[1]).astype(np.int32)
    bins = _be().dmatrix_get_bins(d.handle, 256)
    np.testing.assert_array_equal(hist, oracle.build_hist_fixed(bins, gq, hq, rows=rows))


# 1 row; one CTA, just below / above its minimum; the row count where the grid reaches one CTA per SM, +- 1; several
# overflow windows per CTA
@pytest.mark.parametrize("m", [1, ROWS_PER_CTA - 1, ROWS_PER_CTA + 1, 132 * ROWS_PER_CTA - 1, 132 * ROWS_PER_CTA + 1, 2_400_000])
def test_gathered_histogram_bit_exact(skewed, oracle, m):
    d, b, gpair = skewed
    rows = np.sort(np.random.default_rng(m).choice(gpair.shape[0], size=m, replace=False)).astype(np.uint32)
    gp = gpair[rows]
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gp, mode=MODE_TRAINING_TAIL, row_ids=rows)
    assert kernel == "hist_gather_kernel"
    _check(d, gp, hist, scales, oracle, rows)


@pytest.mark.parametrize("n,F", [(ROWS_PER_CTA - 1, 100), (ROWS_PER_CTA + 1, 104), (300_001, 36), (200_000, 130)])
def test_contiguous_gather_histogram_bit_exact(xgb, oracle, n, F):
    X, y = synth(n, F, 71, "reg")
    rng = np.random.default_rng(3)
    gp = np.stack([rng.standard_normal(n).astype(np.float32), rng.random(n).astype(np.float32) + 0.01], axis=1)
    d = xgb.DMatrix(X, label=y)
    b = xgb.Booster({"max_bin": 256}, [d])
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gp, mode=MODE_FORCE_GATHER)
    assert kernel == "hist_gather_kernel"
    _check(d, gp, hist, scales, oracle, None)


def test_spilling_contiguous_gather_histogram_bit_exact(skewed, oracle):
    d, b, gpair = skewed
    hist, scales, ms, kernel = _be().build_histogram_ex(b.handle, d.handle, gpair, mode=MODE_FORCE_GATHER)
    assert kernel == "hist_gather_kernel"
    _check(d, gpair, hist, scales, oracle, None)


# depth 7 on up to 200k rows: a level's CTA chunks cross many node boundaries, so CTAs flush several segments each
@pytest.mark.parametrize("n,F", [(20000, 28), (200000, 100)])
def test_depth7_trees_bit_exact(xgb, oracle, n, F):
    X, y = synth(n, F, 73, "reg")
    grow_and_compare(xgb, oracle, X, y, dict(objective="reg:squarederror", max_depth=7, eta=0.3, base_score=0.5), 2)


CASES = {
    "sqerr-F100-depth6": (100, dict(objective="reg:squarederror", max_depth=6)),
    "logistic-F100-depth6": (100, dict(objective="binary:logistic", max_depth=6)),
    "sqerr-F104-depth8": (104, dict(objective="reg:squarederror", max_depth=8)),
    "logistic-F104-depth6": (104, dict(objective="binary:logistic", max_depth=6)),
    "sqerr-F8-depth8": (8, dict(objective="reg:squarederror", max_depth=8)),
    "logistic-F36-lossguide": (36, dict(objective="binary:logistic", grow_policy="lossguide", max_leaves=24, max_depth=0)),
    "sqerr-F100-lossguide": (100, dict(objective="reg:squarederror", grow_policy="lossguide", max_leaves=24, max_depth=0)),
    "sqerr-F130-depth6": (130, dict(objective="reg:squarederror", max_depth=6)),
    "logistic-F130-depth8": (130, dict(objective="binary:logistic", max_depth=8)),
}

_TRAIN = r"""
import json, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import sagemaker_xgboost_container_b200 as xgb
from util import synth
be = xgb.get_backend()
for name, (F, extra) in json.loads(sys.argv[2]).items():
    X, y = synth(150000, F, 79, "bin" if "logistic" in name else "reg", quantised=False, missing_frac=0.02)
    d = xgb.DMatrix(X, label=y)
    params = dict(tree_method="hist", max_bin=256, eta=0.3, **extra)
    bst = xgb.train(params, d, num_boost_round=4, verbose_eval=False)
    out = {k: np.asarray(v) for k, v in be.booster_export_model(bst.handle).items()}
    out["cached_margin"] = be.booster_cached_margin(bst.handle, d.handle, 1)
    np.savez("%s/%s.npz" % (sys.argv[3], name), **out)
"""


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    """Every case trained twice, each flush in a process of its own (the switch is read once per process)."""
    out = {}
    for red in (False, True):
        dst = tmp_path_factory.mktemp("red" if red else "partials")
        env = dict(os.environ)
        env.pop("B200XGB_HIST_RED_FLUSH", None)
        if red:
            env["B200XGB_HIST_RED_FLUSH"] = "1"
        r = subprocess.run([sys.executable, "-s", "-c", _TRAIN, ROOT, json.dumps(CASES), str(dst)], capture_output=True, text=True,
                           timeout=900, env=env)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        out[red] = {name: dict(np.load(dst / (name + ".npz"))) for name in CASES}
    return out


@pytest.mark.parametrize("case", sorted(CASES))
def test_models_identical_to_the_red_flush(models, case):
    a, b = models[False][case], models[True][case]
    assert (a["left"] != -1).sum() > 4 * 4, "the trees should really split"
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
