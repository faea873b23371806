"""The predictor against the oracle, bit for bit, on every branch of its plan (run with `pytest -m gpu` on an H100).

Both the device predictor and oracle.predict_margin add fp32 leaf values in tree order to the same fp32 base margin, and
neither is built with fast-math, so margins are compared on their uint32 view and leaf ids exactly: no tolerance.  The
oracle walks the model the device exported (booster_export_model), so this checks the predictor alone, not training.  Each
case first asserts the plan (csrc/predict_plan.h) it means to cover, so a change of plan cannot silently move it to
another branch:
- the tiled kernel with one chunk of trees: 1 ... 300 000 rows (more tiles than CTAs), with and without missing values,
  1 and 3 classes, tree counts of every remainder mod 4 (its 4-trees-at-a-time loop), root-only stumps;
- several chunks: > 96 trained depth-6 trees, the same model with tight node counts after a save / load round trip,
  iteration ranges that begin and end inside chunks;
- 32-row tiles next to full chunks on 900 ... 1247 features;
- thread-per-row for wide rows, for trees beyond the chunk budget, for children that are not adjacent pairs, for matrices
  narrower than the model (dense without NaN, and a libsvm request body), and with B200XGB_PREDICT_LEGACY;
- feature values on and next to every threshold, +-0, +-inf, denormals and NaN; per-row base margins;
- the eval-set prediction cache of a fresh DMatrix and the rmse computed from it.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILED, PER_ROW = "predict_tiled_kernel", "predict_kernel"


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Fitted:
    """A booster, the model it exports (as the oracle reads it) and its class count."""

    def __init__(self, xgb, bst, objective):
        self.bst = bst
        self.m = _be().booster_export_model(bst.handle)
        self.m["objective"] = objective
        self.K = max(1, int(self.m["num_class"]))
        self.rounds = len(self.m["tree_info"]) // self.K
        self.xgb = xgb

    def reload(self, raw):
        return Fitted(self.xgb, self.xgb.Booster(model_file=bytes(raw)), self.m["objective"])

    def plan(self, d, iteration_range=(0, 0)):
        return _be().booster_predict_plan(self.bst.handle, d.handle, iteration_range)

    def check(self, oracle, d, X, iteration_range=(0, 0), base_margin=None):
        """predict(output_margin) and predict(pred_leaf) on d (== X) against the oracle, bit for bit."""
        n = X.shape[0]
        r0, r1 = iteration_range
        tb, te = r0 * self.K, (r1 or self.rounds) * self.K
        margin = self.bst.predict(d, output_margin=True, iteration_range=iteration_range).reshape(n, self.K)
        ref = oracle.predict_margin(self.m, X, tb, te, base_margin=base_margin)
        np.testing.assert_array_equal(_bits(margin), _bits(ref))
        leaf = self.bst.predict(d, pred_leaf=True, iteration_range=iteration_range).reshape(n, te - tb)
        np.testing.assert_array_equal(leaf.astype(np.int32), oracle.predict_leaf(self.m, X, tb, te))
        return margin, leaf


def _train(xgb, params, F, rounds, n=20000, seed=3, K=1, missing_frac=0.1, slots=False):
    """xgb.train returns a copy of the trained booster: its trees are uploaded at their real node counts.  slots=True keeps
    the booster that trained (Booster.update), whose trees stay in the fixed slots of round16(2^(max_depth+1) - 1) nodes
    they were grown in."""
    kind = "multi" if K > 1 else "reg"
    X, y = synth(n, F, seed, kind, K=K, quantised=False, missing_frac=missing_frac)
    params = dict(dict(tree_method="hist", max_bin=256, eta=0.3), **params)
    if K > 1:
        params.update(objective="multi:softprob", num_class=K)
    params.setdefault("objective", "reg:squarederror")
    d = xgb.DMatrix(X, label=y)
    if slots:
        bst = xgb.Booster(params, [d])
        for i in range(rounds):
            bst.update(d, i)
    else:
        bst = xgb.train(params, d, num_boost_round=rounds, verbose_eval=False)
    return Fitted(xgb, bst, params["objective"])


def _slot(max_depth):
    return ((1 << (max_depth + 1)) - 1 + 15) // 16 * 16


def _chunk_sizes(plan):
    return [c["end"] - c["begin"] for c in plan["chunks"]]


# ------------------------------------------------------------------------------------------------------ the models
F_SMALL = 20


@pytest.fixture(scope="module")
def one_chunk(xgb):
    """7 trees of depth 6 (K = 1), 5 rounds x 3 classes of depth 4, and 6 root-only stumps, on 20 features."""
    reg = _train(xgb, dict(max_depth=6), F_SMALL, 7)
    multi = _train(xgb, dict(max_depth=4), F_SMALL, 5, K=3, seed=4)
    stumps = _train(xgb, dict(max_depth=6, gamma=1e30), F_SMALL, 6, seed=5)
    assert (np.diff(stumps.m["tree_offset"]) == 1).all(), "gamma = 1e30 should leave root-only trees"
    return dict(reg=reg, multi=multi, stumps=stumps)


@pytest.fixture(scope="module")
def several_chunks(xgb):
    """The boosters that trained 100 trees of depth 6 (one class) and 60 rounds x 3 classes: the fixed 128-node slots of
    their trees fill a 96 KB chunk at 96 trees."""
    reg = _train(xgb, dict(max_depth=6), 28, 100, n=30000, seed=6, slots=True)
    multi = _train(xgb, dict(max_depth=6), 12, 60, n=30000, K=3, seed=7, slots=True)
    return dict(reg=reg, multi=multi)


# ------------------------------------------------------------------------------------------------------ tiled, one chunk
@pytest.mark.parametrize("has_nan", [False, True])
@pytest.mark.parametrize("n", [1, 1023, 1025, 300_000])
def test_tiled_one_chunk(xgb, oracle, one_chunk, n, has_nan):
    X, _ = synth(n, F_SMALL, 100 + n, "reg", quantised=False, missing_frac=0.2 if has_nan else 0.0)
    d = xgb.DMatrix(X)
    for name, f in one_chunk.items():
        # tree counts 1, 2 and 3 mod 4: whole groups of four traversals plus the remainder loop
        ranges = [(0, 0), (0, f.rounds - 1), (0, f.rounds - 2), (1, f.rounds)]
        for rng in ranges:
            plan = f.plan(d, rng)
            assert plan["kernel"] == TILED and plan["has_nan"] == has_nan and len(plan["chunks"]) == 1, (name, plan)
            assert plan["chunks"][0]["rows"] == 1024
            f.check(oracle, d, X, rng)
    counts = {(f.rounds - r) * f.K % 4 for f in one_chunk.values() for r in (0, 1, 2)}
    assert {1, 2, 3} <= counts


# ------------------------------------------------------------------------------------------------------ several chunks
@pytest.mark.parametrize("has_nan", [False, True])
def test_tiled_several_chunks(xgb, oracle, several_chunks, has_nan):
    reg, multi = several_chunks["reg"], several_chunks["multi"]
    n = 50000
    Xr, _ = synth(n, 28, 200, "reg", quantised=False, missing_frac=0.1 if has_nan else 0.0)
    Xm, _ = synth(n, 12, 201, "reg", quantised=False, missing_frac=0.1 if has_nan else 0.0)
    dr, dm = xgb.DMatrix(Xr), xgb.DMatrix(Xm)
    plan = reg.plan(dr)
    assert plan["kernel"] == TILED and _chunk_sizes(plan) == [96, 4]
    reg.check(oracle, dr, Xr)
    # K = 3: rounds [3, 38) are trees [9, 114): the range starts inside the first chunk of the whole model and ends inside
    # its second; its own chunks are [9, 105) and [105, 114), leaf columns 0 ... 95 and 96 ... 104
    plan = multi.plan(dm, (3, 38))
    assert plan["kernel"] == TILED and [(c["begin"], c["end"]) for c in plan["chunks"]] == [(9, 105), (105, 114)]
    multi.check(oracle, dm, Xm, (3, 38))
    assert _chunk_sizes(multi.plan(dm)) == [96, 84]
    multi.check(oracle, dm, Xm)
    # the same models with tight node counts: saved and loaded, the trees are uploaded at their real sizes
    for f, d, X in ((reg, dr, Xr), (multi, dm, Xm)):
        g = f.reload(f.bst.save_raw("ubj"))
        plan = g.plan(d)
        nodes = np.diff(g.m["tree_offset"])
        assert plan["kernel"] == TILED and sum(c["node_bytes"] for c in plan["chunks"]) == 8 * nodes.sum()
        assert nodes.max() < 128 and len(plan["chunks"]) >= (2 if f is multi else 1), (nodes.mean(), _chunk_sizes(plan))
        np.testing.assert_array_equal(_bits(g.check(oracle, d, X)[0]), _bits(f.bst.predict(d, output_margin=True).reshape(X.shape[0], -1)))
    g = multi.reload(multi.bst.save_raw("ubj"))
    g.check(oracle, dm, Xm, (3, 38))
    g.check(oracle, dm, Xm, (17, 59))


# ------------------------------------------------------------------------------------------------------ 32-row tiles
@pytest.mark.parametrize("F", [900, 1000, 1247])
def test_small_tiles_next_to_full_chunks(xgb, oracle, F):
    """100 depth-6 trees on 900 ... 1247 features: a full chunk leaves room for 32 rows of a tile.  Before chunks were capped
    by that room, F = 1000 and 1247 planned tiles of zero rows (and divided by zero)."""
    f = _train(xgb, dict(max_depth=6), F, 100, n=3000, seed=F, slots=True)
    X, y = synth(5000, F, F + 1, "reg", quantised=False, missing_frac=0.05)
    d = xgb.DMatrix(X, label=y)
    plan = f.plan(d)
    assert plan["kernel"] == TILED and _chunk_sizes(plan) == {900: [96, 4], 1000: [94, 6], 1247: [63, 37]}[F]
    assert all(32 <= c["rows"] for c in plan["chunks"]) and plan["chunks"][0]["rows"] == 32
    assert all(c["smem"] <= 220 * 1024 for c in plan["chunks"])
    f.check(oracle, d, X)
    f.check(oracle, d, X, (10, 99))
    # the eval-set cache of a fresh DMatrix is brought up to date by the same plan
    cache = _be().booster_cached_margin(f.bst.handle, d.handle, 1)
    np.testing.assert_array_equal(_bits(cache), _bits(oracle.predict_margin(f.m, X)))


# ------------------------------------------------------------------------------------------------------ thread-per-row
def test_thread_per_row_for_wide_rows(xgb, oracle):
    f = _train(xgb, dict(max_depth=6), 1300, 10, n=3000, seed=8)
    X, _ = synth(4000, 1300, 9, "reg", quantised=False, missing_frac=0.05)
    d = xgb.DMatrix(X)
    plan = f.plan(d)
    assert plan["kernel"] == PER_ROW and plan["reason"] == "rows too wide"
    f.check(oracle, d, X)
    f.check(oracle, d, X, (3, 7))


def test_thread_per_row_for_trees_beyond_the_chunk_budget(xgb, oracle):
    """max_depth = 13: a trained tree's slot holds 16384 nodes, 128 KB, more than a chunk."""
    f = _train(xgb, dict(max_depth=13, min_child_weight=0.5), 16, 3, n=40000, seed=10, slots=True)
    X, _ = synth(30000, 16, 11, "reg", quantised=False, missing_frac=0.1)
    d = xgb.DMatrix(X)
    plan = f.plan(d)
    assert _slot(13) * 8 > 96 * 1024
    assert plan["kernel"] == PER_ROW and plan["reason"] == "tree too large"
    assert (f.m["left"] != -1).sum() > 3 * 1000, "the trees should be deep"
    f.check(oracle, d, X)
    f.check(oracle, d, X, (1, 3))


def _preorder(tree):
    """Renumber one tree of a JSON model in depth-first pre-order: a left child follows its parent, the right child
    follows the left subtree, so siblings stop being adjacent pairs."""
    L, R = tree["left_children"], tree["right_children"]
    order, stack = [], [0]
    while stack:
        i = stack.pop()
        order.append(i)
        if L[i] != -1:
            stack += [R[i], L[i]]
    new = {old: k for k, old in enumerate(order)}
    for key in ("base_weights", "default_left", "loss_changes", "split_conditions", "split_indices", "split_type", "sum_hessian"):
        tree[key] = [tree[key][i] for i in order]
    tree["left_children"] = [new[L[i]] if L[i] != -1 else -1 for i in order]
    tree["right_children"] = [new[R[i]] if R[i] != -1 else -1 for i in order]
    tree["parents"] = [2147483647] + [0] * (len(order) - 1)
    for k, i in enumerate(order):
        if L[i] != -1:
            tree["parents"][new[L[i]]] = tree["parents"][new[R[i]]] = k


def test_children_not_adjacent(xgb, oracle, one_chunk, several_chunks):
    for f in (one_chunk["reg"], one_chunk["multi"], several_chunks["reg"]):
        doc = json.loads(bytes(f.bst.save_raw("json")))
        for t in doc["learner"]["gradient_booster"]["model"]["trees"]:
            _preorder(t)
        g = f.reload(json.dumps(doc).encode())
        internal = g.m["left"] != -1
        assert (g.m["right"][internal] != g.m["left"][internal] + 1).any()
        F = int(g.bst.num_features())
        X, _ = synth(20000, F, 12, "reg", quantised=False, missing_frac=0.1)
        d = xgb.DMatrix(X)
        plan = g.plan(d)
        assert plan["kernel"] == PER_ROW and plan["reason"] == "children not adjacent"
        g.check(oracle, d, X)
        # the same trees renumbered: same margins as the original model
        np.testing.assert_array_equal(_bits(g.bst.predict(d, output_margin=True)), _bits(f.bst.predict(d, output_margin=True)))


# ------------------------------------------------------------------------------------------------------ narrow matrices
def test_matrix_narrower_than_the_model(xgb, oracle, one_chunk, several_chunks):
    """A dense matrix without the model's last 3 features and no NaN: the missing features are missing values (default
    direction), not the pad column or the next row's values."""
    for f in (one_chunk["reg"], one_chunk["multi"], several_chunks["reg"]):
        F = int(f.bst.num_features())
        assert (f.m["split_index"][f.m["left"] != -1] >= F - 3).any(), "the model should split on the last features"
        X, _ = synth(5000, F, 13, "reg", quantised=False)
        Xn = np.ascontiguousarray(X[:, :F - 3])
        d = xgb.DMatrix(Xn)
        plan = f.plan(d)
        assert plan["kernel"] == PER_ROW and plan["reason"] == "matrix narrower than the model" and not plan["has_nan"]
        f.check(oracle, d, Xn)
        # the wide matrix with those features missing predicts the same
        Xw = X.copy()
        Xw[:, F - 3:] = np.nan
        np.testing.assert_array_equal(_bits(f.bst.predict(d, output_margin=True)), _bits(f.bst.predict(xgb.DMatrix(Xw), output_margin=True)))


def test_libsvm_request_body_narrower_than_the_model(xgb, oracle, one_chunk):
    """serving.sparse_libsvm_to_dmatrix sizes the matrix by the largest index in the body: a body that never names the
    model's last features gives a matrix narrower than the model."""
    from sagemaker_xgboost_container_b200 import serving
    f = one_chunk["reg"]
    F = int(f.bst.num_features())
    rng = np.random.default_rng(14)
    n, width = 3000, F - 4
    X = np.full((n, width), np.nan, np.float32)
    lines = []
    for r in range(n):
        cols = np.sort(rng.choice(width, size=int(rng.integers(1, width + 1)), replace=False))
        cols[-1] = width - 1 if r == 0 else cols[-1]           # one row names the last column: the matrix is `width` wide
        vals = rng.standard_normal(len(cols)).astype(np.float32)
        X[r, cols] = vals
        lines.append(" ".join("%d:%r" % (c, float(v)) for c, v in zip(cols, vals)))
    d = serving.sparse_libsvm_to_dmatrix("\n".join(lines))
    assert d.num_col() == width and d.num_row() == n
    Xd = _be().dmatrix_get_raw(d.handle).reshape(n, width)        # the values as parsed on the device
    np.testing.assert_array_equal(np.isnan(Xd), np.isnan(X))
    np.testing.assert_allclose(Xd, X, rtol=1e-7)
    plan = f.plan(d)
    assert plan["kernel"] == PER_ROW and plan["reason"] == "matrix narrower than the model"
    f.check(oracle, d, Xd)


# ------------------------------------------------------------------------------------------------------ comparison edges
def _edge_model(xgb, f):
    """f's trees with some thresholds moved to 0, -0, +-the smallest denormal and the smallest normal."""
    doc = json.loads(bytes(f.bst.save_raw("json")))
    special = [0.0, -0.0, 1.401298464324817e-45, -1.401298464324817e-45, 1.1754943508222875e-38]
    k = 0
    for t in doc["learner"]["gradient_booster"]["model"]["trees"]:
        for i, l in enumerate(t["left_children"]):
            if l != -1 and i % 3 == 0:
                t["split_conditions"][i] = special[k % len(special)]
                k += 1
    g = f.reload(json.dumps(doc).encode())
    cond = g.m["split_cond"][g.m["left"] != -1]
    assert k >= 10 and (np.signbit(cond) & (cond == 0)).any() and ((cond != 0) & (np.abs(cond) < 1.1754944e-38)).any()
    return g


@pytest.mark.parametrize("has_nan", [False, True])
def test_values_on_and_next_to_every_threshold(xgb, oracle, one_chunk, has_nan):
    specials = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754944e-38, -1.1754944e-38], np.float32)
    for f in (_edge_model(xgb, one_chunk["reg"]), one_chunk["multi"]):
        m = f.m
        internal = m["left"] != -1
        F = int(f.bst.num_features())
        rng = np.random.default_rng(15)
        n = 40000
        X = np.empty((n, F), np.float32)
        for j in range(F):
            c = m["split_cond"][internal & (m["split_index"] == j)].astype(np.float32)
            pool = np.concatenate([c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf)), specials])
            if has_nan:
                pool = np.append(pool, np.float32(np.nan))
            X[:, j] = rng.choice(pool, size=n)
        d = xgb.DMatrix(X)
        plan = f.plan(d)
        assert plan["kernel"] == TILED and plan["has_nan"] == has_nan
        f.check(oracle, d, X)


# ------------------------------------------------------------------------------------------------------ base margins
@pytest.mark.parametrize("which", ["reg", "multi"])
def test_per_row_base_margin(xgb, oracle, one_chunk, several_chunks, which):
    for f, F in ((one_chunk[which], F_SMALL), (several_chunks[which], 28 if which == "reg" else 12)):
        n = 4097
        X, _ = synth(n, F, 16, "reg", quantised=False, missing_frac=0.1)
        bm = np.random.default_rng(17).standard_normal((n, f.K)).astype(np.float32) * 3
        d = xgb.DMatrix(X, base_margin=bm.ravel() if f.K > 1 else bm[:, 0])
        assert f.plan(d)["kernel"] == TILED
        f.check(oracle, d, X, base_margin=bm)
        f.check(oracle, d, X, (1, f.rounds - 1), base_margin=bm)


# ------------------------------------------------------------------------------------------------------ legacy kernel
_LEGACY = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import sagemaker_xgboost_container_b200 as xgb
be = xgb.get_backend()
inp = np.load(sys.argv[2])
out = {}
for i in range(int(inp["count"])):
    bst = xgb.Booster(model_file=bytes(inp["model%d" % i]))
    d = xgb.DMatrix(inp["X%d" % i])
    plan = be.booster_predict_plan(bst.handle, d.handle)
    assert plan["kernel"] == "predict_kernel" and plan["reason"] == "B200XGB_PREDICT_LEGACY", plan
    out["margin%d" % i] = bst.predict(d, output_margin=True)
    out["leaf%d" % i] = bst.predict(d, pred_leaf=True)
    out["range%d" % i] = bst.predict(d, output_margin=True, iteration_range=(1, bst.num_boosted_rounds() - 1))
np.savez(sys.argv[3], **out)
"""


def test_legacy_kernel_gives_the_same_bits(xgb, tmp_path, one_chunk, several_chunks):
    """B200XGB_PREDICT_LEGACY=1 (read once per process, so in a subprocess) runs the thread-per-row kernel: the same bits
    as the tiled kernel on a one-chunk, a multi-chunk and a 3-class model."""
    cases = [one_chunk["reg"], several_chunks["reg"], several_chunks["multi"]]
    inp = {"count": len(cases)}
    here = []
    for i, f in enumerate(cases):
        F = int(f.bst.num_features())
        X, _ = synth(20000, F, 18 + i, "reg", quantised=False, missing_frac=0.1 if i != 1 else 0.0)
        raw = bytes(f.bst.save_raw("ubj"))
        inp["model%d" % i], inp["X%d" % i] = np.frombuffer(raw, np.uint8), X
        d = xgb.DMatrix(X)
        assert f.plan(d)["kernel"] == TILED and len(f.plan(d)["chunks"]) == (1 if i == 0 else 2)
        here.append((f.bst.predict(d, output_margin=True), f.bst.predict(d, pred_leaf=True),
                     f.bst.predict(d, output_margin=True, iteration_range=(1, f.rounds - 1))))
    np.savez(tmp_path / "in.npz", **inp)
    env = dict(os.environ, B200XGB_PREDICT_LEGACY="1")
    r = subprocess.run([sys.executable, "-s", "-c", _LEGACY, ROOT, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = np.load(tmp_path / "out.npz")
    for i, (margin, leaf, part) in enumerate(here):
        np.testing.assert_array_equal(_bits(out["margin%d" % i]), _bits(margin))
        np.testing.assert_array_equal(out["leaf%d" % i], leaf)
        np.testing.assert_array_equal(_bits(out["range%d" % i]), _bits(part))


# ------------------------------------------------------------------------------------------------------ eval cache
def test_eval_set_on_a_fresh_matrix(xgb, oracle, several_chunks):
    """Multi-chunk models evaluated on a fresh DMatrix, one loaded (tight node counts) and the booster that trained (slots):
    the prediction cache is filled by the predictor (bit-exact), and rmse over it (squares in fp32, sums in double) matches
    numpy over the oracle's margins."""
    loaded = _train(xgb, dict(max_depth=6), 28, 200, n=30000, seed=6)
    loaded = loaded.reload(loaded.bst.save_raw("ubj"))
    X, y = synth(70000, 28, 19, "reg", quantised=False, missing_frac=0.05)
    for f in (loaded, several_chunks["reg"]):
        f.bst.set_param({"eval_metric": "rmse"})
        d = xgb.DMatrix(X, label=y)
        assert len(f.plan(d)["chunks"]) >= 2
        msg = f.bst.eval_set([(d, "eval")])
        value = float(msg.split("eval-rmse:")[1].split()[0])
        ref = oracle.predict_margin(f.m, X)
        np.testing.assert_array_equal(_bits(_be().booster_cached_margin(f.bst.handle, d.handle, 1)), _bits(ref))
        diff = ref[:, 0] - y
        expect = np.sqrt(np.sum((diff * diff).astype(np.float64)) / len(y))
        assert abs(value - expect) <= 1e-6 * expect, (value, expect)
