"""QuantileDMatrix and DataIter on the GPU (run with `pytest -m gpu` on an H100): cuts and every binned copy against DMatrix,
XGB200DMatrixRankCuts and tests/cuts_reference.py bit for bit; models trained on several batches against DMatrix models byte
for byte; the bin predictor against the float predictor on both launch plans; a foreign model against a numpy restatement of
the lower-edge rule; eval sets, early stopping and resuming; the engine's peak device bytes; and every error."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cuts_reference as R
from util import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _be():
    from sagemaker_xgboost_container_b200.backend import get_backend
    return get_backend()


def _u32(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _iter(xgb, batches, device=False):
    """A DataIter over a list of dicts (data, label, ...), recording its calls; device=True yields data as torch CUDA tensors."""

    class It(xgb.DataIter):
        def __init__(self):
            super().__init__()
            self.i, self.calls = 0, []

        def reset(self):
            self.calls.append("reset")
            self.i = 0

        def next(self, input_data):
            self.calls.append("next")
            if self.i == len(batches):
                return False
            b = dict(batches[self.i])
            if device:
                import torch
                b["data"] = torch.from_numpy(np.ascontiguousarray(b["data"])).cuda()
            input_data(**b)
            self.i += 1
            return True

    return It()


def _split(bounds, X, **meta):
    out = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        d = {"data": X[a:b]}
        for k, v in meta.items():
            if v is not None:
                d[k] = v[a:b]
        out.append(d)
    return out


def _cuts(d):
    return _be().dmatrix_get_cuts(d.handle, 256)


def _assert_same_cuts(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(_u32(got[1]), _u32(want[1]))
    np.testing.assert_array_equal(_u32(got[2]), _u32(want[2]))


def _assert_same_bins(dq, dd):
    be = _be()
    _assert_same_cuts(_cuts(dq), _cuts(dd))
    assert _cuts(dq)[3] == _cuts(dd)[3], "has_missing differs"
    np.testing.assert_array_equal(be.dmatrix_get_bins(dq.handle, 256), be.dmatrix_get_bins(dd.handle, 256))
    (aq, cq), (ad, cd) = be.dmatrix_get_bin_copies(dq.handle, 256), be.dmatrix_get_bin_copies(dd.handle, 256)
    assert (aq is None) == (ad is None)
    if aq is not None:
        np.testing.assert_array_equal(aq, ad)
    np.testing.assert_array_equal(cq, cd)


# ------------------------------------------------------------------------------------------------ one batch
@pytest.mark.parametrize("source", ["numpy", "pandas", "csr", "torch"])
@pytest.mark.parametrize("kind", ["continuous", "missing-999"])
def test_one_batch_is_dmatrix(xgb, source, kind):
    """One batch takes the exact single-rank cuts: cuts and all binned copies equal DMatrix on the same data (F = 100: main,
    4-wide tail, aligned copy), above the summary cap, and the caller's array is left as it was.  A CSR matrix marks missing
    values by absence and keeps its stored values whatever `missing` says, as DMatrix(csr) does."""
    rng = np.random.default_rng(7)
    n, F = 5000, 100
    X = rng.standard_normal((n, F)).astype(f32)
    missing = None
    if kind == "missing-999":
        X[rng.random((n, F)) < 0.05] = -999.0
        missing = -999.0
    if source == "csr":
        import scipy.sparse as sp
        X[rng.random((n, F)) < 0.3] = 0.0
        data = sp.csr_matrix(X)
        dd = xgb.DMatrix(data)                                      # stored values stay values, whatever `missing` says
    elif source == "pandas":
        import pandas as pd
        data = pd.DataFrame(X, columns=["c%d" % i for i in range(F)])
        dd = xgb.DMatrix(X, missing=missing)
    elif source == "torch":
        import torch
        data = torch.from_numpy(X.copy()).cuda()
        dd = xgb.DMatrix(X, missing=missing)
    else:
        data = X
        dd = xgb.DMatrix(X, missing=missing)
    before = X.copy()
    dq = xgb.QuantileDMatrix(data, missing=missing)
    assert dq.num_row() == n and dq.num_col() == F
    _assert_same_bins(dq, dd)
    after = data.cpu().numpy() if source == "torch" else (data.toarray() if source == "csr" else np.asarray(data, f32))
    np.testing.assert_array_equal(_u32(after), _u32(before))
    if source == "pandas":
        assert dq.feature_names == list(data.columns)


# ------------------------------------------------------------------------------------------------ several batches
@pytest.mark.parametrize("above_cap", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_several_batches_cuts(xgb, above_cap, weighted):
    """Several batches: the multi-rank recipe over the batches' row ranges, bit for bit against XGB200DMatrixRankCuts and
    cuts_reference.rank_cuts; below the cap (quantised data) the DMatrix cuts as well.  The bins follow the cuts."""
    n, F = 7500, 100
    X, _ = synth(n, F, 11, quantised=not above_cap, missing_frac=0.02)
    w = np.random.default_rng(3).integers(1, 5, n).astype(f32) if weighted else None
    bounds = [0, 2500, 4100, 7500]
    it = _iter(xgb, _split(bounds, X, weight=w))
    dq = xgb.QuantileDMatrix(it)
    assert it.calls == ["reset"] + ["next"] * 4 + ["reset"] + ["next"] * 4
    dd = xgb.DMatrix(X, weight=w)
    got = _cuts(dq)
    _assert_same_cuts(got, _be().dmatrix_rank_cuts(dd.handle, 256, bounds))
    _assert_same_cuts(got, R.rank_cuts(X, 256, bounds, w))
    assert got[3]
    if not above_cap:
        assert R.in_exact_regime(w, n)
        _assert_same_bins(dq, dd)
    np.testing.assert_array_equal(_be().dmatrix_get_bins(dq.handle, 256), R.bin_matrix(X, got[0], got[1]))
    np.testing.assert_array_equal(dq.get_weight(), w if weighted else np.zeros(0, f32))


# ------------------------------------------------------------------------------------------------ training
N, FT = 6000, 20
BOUNDS = [0, 1700, 2900, 6000]


def _family(name):
    X, y = synth(N, FT, 21, "bin" if name == "binary:logistic" else ("multi" if name == "multi:softprob" else "reg"), K=3)
    meta, params = {"label": y}, {"objective": name, "max_depth": 5, "eta": 0.3}
    if name == "multi:softprob":
        params["num_class"] = 3
    elif name == "reg:quantileerror":
        params["quantile_alpha"] = "(0.1,0.5,0.9)"
    elif name == "survival:aft":
        lo = np.exp(y).astype(f32)
        hi = np.where(np.arange(N) % 3 == 0, np.inf, lo).astype(f32)
        meta = {"label_lower_bound": lo, "label_upper_bound": hi}
    elif name == "rank:ndcg":
        meta = {"label": np.clip(np.round(y + 1.5), 0, 3).astype(f32), "qid": np.arange(N) // 7}    # groups of 7 cross the batch bounds
    elif name == "lossguide":
        params = {"objective": "reg:squarederror", "grow_policy": "lossguide", "max_leaves": 24, "max_depth": 0, "eta": 0.3}
    elif name == "monotone":
        params = {"objective": "reg:squarederror", "monotone_constraints": "(" + ",".join(["1", "-1"] + ["0"] * (FT - 2)) + ")", "max_depth": 5}
    elif name == "gradient_based":
        params = {"objective": "reg:squarederror", "sampling_method": "gradient_based", "subsample": 0.5, "max_depth": 5}
    return X, meta, params


FAMILIES = ["reg:squarederror", "binary:logistic", "multi:softprob", "reg:absoluteerror", "reg:quantileerror", "survival:aft", "rank:ndcg",
            "lossguide", "monotone", "gradient_based"]


@pytest.mark.parametrize("name", FAMILIES)
def test_training_equals_dmatrix(xgb, name):
    """Data below the cap: a model trained on a three-batch QuantileDMatrix is the DMatrix model byte for byte."""
    X, meta, params = _family(name)
    dq = xgb.QuantileDMatrix(_iter(xgb, _split(BOUNDS, X, **meta)))
    dd = xgb.DMatrix(X, **meta)
    if "qid" in meta:
        np.testing.assert_array_equal(dq.get_uint_info("group_ptr"), dd.get_uint_info("group_ptr"))
    a = xgb.train(params, dq, num_boost_round=5, verbose_eval=False)
    b = xgb.train(params, dd, num_boost_round=5, verbose_eval=False)
    assert bytes(a.save_raw("ubj")) == bytes(b.save_raw("ubj"))


# ------------------------------------------------------------------------------------------------ prediction
def _same_predictions(bst, dq, dd, K, iteration_range=(0, 0)):
    for kw in ({"output_margin": True}, {}, {"pred_leaf": True}):
        p, q = bst.predict(dq, iteration_range=iteration_range, **kw), bst.predict(dd, iteration_range=iteration_range, **kw)
        assert p.shape == q.shape
        np.testing.assert_array_equal(_u32(p), _u32(q))


def _pred_data(n, F, seed, K):
    """quantised rows with 5 % missing; the label leans on the last two features, so the trees split on the tail block"""
    X, y = synth(n, F, seed, "multi" if K > 1 else "reg", K=K, missing_frac=0.05)
    a, b = np.nan_to_num(X[:, F - 1]), np.nan_to_num(X[:, F - 2])
    y = ((a > 0).astype(f32) + (b > 0.5)).astype(f32) if K > 1 else (y + 2 * a + b).astype(f32)
    return X, y


# The tiled bin kernel stages rows four ways: F = 20 (one padded group, no tail, packed rows), 36 (4-byte tail from bins_tail,
# packed rows), 72 (8-byte tail from bins_tail, packed rows), 100 (aligned 128 B rows, 4-byte tail from bins_tail) and 104
# (aligned rows holding the 8-byte tail).  F = 5100 stages no rows: too wide, the thread-per-row kernel runs.
@pytest.mark.parametrize("F,plan,aligned", [(20, "predict_bins_tiled_kernel", False), (36, "predict_bins_tiled_kernel", False),
                                            (72, "predict_bins_tiled_kernel", False), (100, "predict_bins_tiled_kernel", True),
                                            (104, "predict_bins_tiled_kernel", True), (5100, "predict_bins_kernel", False)])
@pytest.mark.parametrize("K", [1, 3])
def test_bin_predictor_equals_float_predictor(xgb, tmp_path, F, plan, aligned, K):
    """Margins, values and leaves from the bins equal the float predictor's bits: on the training matrix, on an eval matrix
    built on its cuts (ref=), with iteration_range and base_margin, and for a model loaded from a file that was trained on a
    DMatrix with the same cuts, for every way the tiled kernel stages a row and for the thread-per-row kernel."""
    n = 3000 if F > 1000 else 8000
    X, y = _pred_data(n, F, 5, K)
    params = {"objective": "multi:softprob", "num_class": K} if K > 1 else {"objective": "reg:squarederror"}
    params.update(max_depth=6, eta=0.3)
    bounds = [0, n // 3, n]
    dq = xgb.QuantileDMatrix(_iter(xgb, _split(bounds, X, label=y)))
    dd = xgb.DMatrix(X, label=y)
    assert (_be().dmatrix_get_bin_copies(dq.handle, 256)[0] is not None) == aligned
    bst = xgb.train(params, dq, num_boost_round=6, verbose_eval=False)
    got = _be().booster_predict_plan(bst.handle, dq.handle)
    assert got["kernel"] == plan, got
    if F % 32:                                                     # the model reads the last group or the tail
        assert (_be().booster_export_model(bst.handle)["split_index"] >= F // 32 * 32).any()
    _same_predictions(bst, dq, dd, K)
    _same_predictions(bst, dq, dd, K, iteration_range=(2, 5))
    Xv, yv = _pred_data(2000, F, 6, K)
    bm = np.random.default_rng(1).standard_normal((2000, K)).astype(f32).reshape(-1) * 0.1
    dqv = xgb.QuantileDMatrix(Xv, label=yv, ref=dq, base_margin=bm)
    ddv = xgb.DMatrix(Xv, label=yv, base_margin=bm)
    _same_predictions(bst, dqv, ddv, K)
    path = str(tmp_path / "m.json")
    xgb.train(params, dd, num_boost_round=4, verbose_eval=False).save_model(path)
    loaded = xgb.Booster(model_file=path)
    _same_predictions(loaded, dq, dd, K)


def _lower_edge_walk(m, X_edge, n_trees):
    """leaf ids and fp32 margins of the exported model on X_edge, every tree at weight 1, in tree order"""
    n = X_edge.shape[0]
    leaves = np.zeros((n, n_trees), np.int32)
    margin = np.full(n, m["base_score"], f32)
    rows = np.arange(n)
    for t in range(n_trees):
        o = m["tree_offset"][t]
        nid = np.zeros(n, np.int64)
        while True:
            inner = m["left"][o + nid] != -1
            if not inner.any():
                break
            f = m["split_index"][o + nid]
            v = X_edge[rows, f]
            go_left = np.where(np.isnan(v), m["default_left"][o + nid] != 0, v < m["split_cond"][o + nid])
            nid = np.where(inner, np.where(go_left, m["left"][o + nid], m["right"][o + nid]), nid)
        leaves[:, t] = nid
        margin = (margin + m["split_cond"][o + nid]).astype(f32)
    return leaves, margin


def test_foreign_model_lower_edge_rule(xgb):
    """A model whose thresholds are not cut values of the matrix: the bin predictor equals a numpy walk of the model over
    each value replaced by its bin's lower edge (min_vals for bin 0, missing stays missing)."""
    Xa, ya = synth(4000, 12, 31, quantised=False)
    bst = xgb.train({"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.25}, xgb.DMatrix(Xa, label=ya), num_boost_round=8, verbose_eval=False)
    X, _ = synth(5000, 12, 32, missing_frac=0.05)
    dq = xgb.QuantileDMatrix(X)
    ptrs, vals, mins, _ = _cuts(dq)
    b = _be().dmatrix_get_bins(dq.handle, 256).reshape(X.shape).astype(np.int64)
    Xe = np.empty_like(X)
    for f in range(X.shape[1]):
        edges = np.concatenate([[mins[f]], vals[ptrs[f]:ptrs[f + 1] - 1]]).astype(f32)
        Xe[:, f] = np.where(b[:, f] == 255, np.nan, edges[np.minimum(b[:, f], len(edges) - 1)])
    m = _be().booster_export_model(bst.handle)
    leaves, margin = _lower_edge_walk(m, Xe, 8)
    np.testing.assert_array_equal(bst.predict(dq, pred_leaf=True).astype(np.int32), leaves)
    np.testing.assert_array_equal(_u32(bst.predict(dq, output_margin=True)), _u32(margin))


# ------------------------------------------------------------------------------------------------ evals and resuming
def test_eval_sets_early_stopping_and_resume(xgb):
    X, y = synth(6000, 16, 41, "bin")
    Xv, yv = synth(3000, 16, 42, "bin")
    params = {"objective": "binary:logistic", "max_depth": 5, "eta": 0.5, "eval_metric": ["logloss", "auc"]}
    dq = xgb.QuantileDMatrix(_iter(xgb, _split([0, 2000, 6000], X, label=y)))
    dqv = xgb.QuantileDMatrix(_iter(xgb, _split([0, 1000, 3000], Xv, label=yv)), ref=dq)
    dd, ddv = xgb.DMatrix(X, label=y), xgb.DMatrix(Xv, label=yv)
    rq, rd = {}, {}
    a = xgb.train(params, dq, 40, evals=[(dq, "train"), (dqv, "val")], evals_result=rq, early_stopping_rounds=3, verbose_eval=False)
    b = xgb.train(params, dd, 40, evals=[(dd, "train"), (ddv, "val")], evals_result=rd, early_stopping_rounds=3, verbose_eval=False)
    assert rq == rd and a.best_iteration == b.best_iteration
    assert bytes(a.save_raw("ubj")) == bytes(b.save_raw("ubj"))
    a2 = xgb.train(params, dq, 3, xgb_model=xgb.train(params, dq, 3, verbose_eval=False), verbose_eval=False)
    b2 = xgb.train(params, dd, 3, xgb_model=xgb.train(params, dd, 3, verbose_eval=False), verbose_eval=False)
    assert bytes(a2.save_raw("ubj")) == bytes(b2.save_raw("ubj"))


# ------------------------------------------------------------------------------------------------ memory
def test_peak_engine_bytes_from_device_batches(xgb):
    """Built from torch CUDA batches, the engine's peak bytes stay below the binned copies + one batch + the summary scratch,
    and below n x F x 4 (the float matrix a DMatrix would hold)."""
    nb, rows, F = 8, 100_000, 100
    batches = [{"data": synth(rows, F, 100 + i)[0]} for i in range(nb)]
    n = nb * rows
    be = _be()
    live0, _ = be.device_memory(reset_peak=True)
    dq = xgb.QuantileDMatrix(_iter(xgb, batches, device=True))
    live1, peak = be.device_memory()
    binned = (n + 512) * (96 + 4) + n * 128 + 128 + n * F          # main + tail (with pad rows), aligned copy, column-major copy
    one_batch = rows * F * 4
    summary = rows * 4 * 6 + (1 << 20)                               # keys x2, values, counts, weights x2 + CUB temp
    assert live1 - live0 <= binned + (1 << 20)
    assert peak - live0 <= binned + one_batch + summary, (peak - live0, binned, one_batch, summary)
    assert peak - live0 < n * F * 4
    del dq


# ------------------------------------------------------------------------------------------------ errors
def _raises(xgb, fn, *words):
    with pytest.raises(xgb.XGBoostError) as e:
        fn()
    for w in words:
        assert w in str(e.value), str(e.value)


def test_errors(xgb):
    X, y = synth(3000, 10, 51)
    dq = xgb.QuantileDMatrix(_iter(xgb, _split([0, 1000, 3000], X, label=y)))
    bst = xgb.train({"max_depth": 3}, dq, 2, verbose_eval=False)
    _raises(xgb, lambda: bst.predict(dq, pred_contribs=True), "QuantileDMatrix", "pred_contribs")
    _raises(xgb, lambda: xgb.train({"booster": "dart", "rate_drop": 0.1}, dq, 2, verbose_eval=False), "QuantileDMatrix", "dart")
    dart = xgb.train({"booster": "dart", "rate_drop": 0.1}, xgb.DMatrix(X, label=y), 2, verbose_eval=False)
    _raises(xgb, lambda: dart.predict(dq), "QuantileDMatrix", "dart")
    _raises(xgb, lambda: xgb.train({"process_type": "update", "updater": "refresh"}, dq, 2, xgb_model=bst, verbose_eval=False),
            "QuantileDMatrix", "process_type=update")
    _raises(xgb, lambda: dq.slice([0, 1, 2]), "QuantileDMatrix", "slice")
    _raises(xgb, lambda: xgb.cv({"max_depth": 3}, dq, 2, nfold=2), "QuantileDMatrix", "slice")
    _raises(xgb, lambda: _be().dmatrix_get_raw(dq.handle), "QuantileDMatrix", "XGB200DMatrixGetRaw")
    p, v, m, _ = _cuts(dq)
    _raises(xgb, lambda: _be().dmatrix_set_cuts(dq.handle, p, v, m), "QuantileDMatrix", "XGB200DMatrixSetCuts")
    _raises(xgb, lambda: xgb.train({"max_bin": 64}, dq, 1, verbose_eval=False), "max_bin")
    d64 = xgb.QuantileDMatrix(X, label=y, max_bin=64)
    xgb.train({"max_bin": 64}, d64, 1, verbose_eval=False)
    dq.set_weight(np.full(3000, 2.0, f32))                         # new weights keep the cuts, training reads them
    _assert_same_cuts(_cuts(dq), R.rank_cuts(X, 256, [0, 1000, 3000]))
    xgb.train({"max_depth": 3}, dq, 1, verbose_eval=False)
    with pytest.raises(xgb.XGBoostError):
        xgb.DMatrix(_iter(xgb, []))


def test_batches_must_repeat(xgb):
    X, y = synth(3000, 10, 52)

    class Shrinking(xgb.DataIter):
        def __init__(self, second):
            super().__init__()
            self.passes, self.i, self.second = 0, 0, second

        def reset(self):
            self.passes += 1
            self.i = 0

        def next(self, input_data):
            if self.i == 2:
                return False
            a, b = (0, 1000) if self.i == 0 else (1000, 3000)
            if self.passes == 2 and self.second == "rows" and self.i == 1:
                b -= 1
            cols = 9 if (self.second == "cols" and self.i == 1) else 10
            input_data(data=X[a:b, :cols], label=y[a:b])
            self.i += 1
            return True

    _raises(xgb, lambda: xgb.QuantileDMatrix(Shrinking("rows")), "second pass")
    _raises(xgb, lambda: xgb.QuantileDMatrix(Shrinking("cols")), "columns")


def test_missing_values_against_full_ref_cuts(xgb):
    """ref cuts that use all 256 codes leave no code for missing values: an eval matrix with missing values raises by name."""
    rng = np.random.default_rng(60)
    X = rng.standard_normal((5000, 4)).astype(f32)
    dtrain = xgb.QuantileDMatrix(X)
    assert int(np.diff(_cuts(dtrain)[0]).max()) == 256
    Xv = X[:100].copy()
    Xv[0, 0] = np.nan
    _raises(xgb, lambda: xgb.QuantileDMatrix(Xv, ref=dtrain), "missing values", "256")
    xgb.QuantileDMatrix(X[:100], ref=dtrain)
    Xm = X.copy()
    Xm[::50, 1] = np.nan
    dm = xgb.QuantileDMatrix(Xm, label=X[:, 2])                    # with missing values of its own: 255 codes, eval sets with NaN work
    dv = xgb.QuantileDMatrix(Xv, label=X[:100, 2], ref=dm)
    bst = xgb.train({"max_depth": 4}, dm, 2, evals=[(dv, "v")], verbose_eval=False)
    np.testing.assert_array_equal(_u32(bst.predict(dv)), _u32(bst.predict(xgb.DMatrix(Xv))))


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_ranks_raise(tmp_path):
    """Under a communicator with world_size > 1 a QuantileDMatrix raises by name."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "err")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           "29631", os.path.join(ROOT, "tests", "helpers", "quantile_dmatrix_shard_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    with open(out) as f:
        assert "QuantileDMatrix is not supported with more than one GPU" in f.read()
