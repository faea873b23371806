"""The host side of QuantileDMatrix without a GPU: how core.QuantileDMatrix drives a DataIter and hands each batch to the
engine, checked against a stand-in backend that iterates like the engine (reset, next until False, twice).  The engine's own
checks (shapes between passes, meta lengths, cuts) are covered on the GPU in test_gpu_quantile_dmatrix.py."""
import numpy as np
import pytest

import sagemaker_xgboost_container_b200 as xgb
from sagemaker_xgboost_container_b200 import core


class FakeEngine:
    """Records the proxy calls of every pass; a pass is reset() then next() until it returns False."""

    supports_ranking = True

    def __init__(self):
        self.passes, self.freed = [], []

    def proxy_create(self):
        return "proxy"

    def proxy_set_dense(self, h, arr):
        self.passes[-1].append({"kind": "dense", "shape": arr.shape, "dtype": arr.dtype.str})

    def proxy_set_cuda(self, h, obj):  # pragma: no cover - no device here
        raise AssertionError("no device batches in these tests")

    def proxy_set_csr(self, h, indptr, indices, data, ncol):
        self.passes[-1].append({"kind": "csr", "rows": len(indptr) - 1, "ncol": ncol, "dtypes": (indptr.dtype.str, indices.dtype.str, data.dtype.str)})

    def dmatrix_set_info_interface(self, h, field, arr):
        self.passes[-1][-1][field] = np.array(arr)

    def quantile_dmatrix_from_callback(self, proxy, ref, reset, next_, missing, max_bin):
        self.max_bin, self.missing = max_bin, missing
        for _ in range(2):
            self.passes.append(["reset"])
            reset()
            while True:
                self.passes[-1].append("next")
                if not next_():
                    break
        return "qdm"

    def dmatrix_free(self, h):
        self.freed.append(h)

    def dmatrix_num_col(self, h):
        return 3

    def dmatrix_set_str_info(self, h, field, values):
        self.str_info = (field, list(values))


@pytest.fixture
def engine(monkeypatch):
    e = FakeEngine()
    monkeypatch.setattr(core, "get_backend", lambda: e)
    return e


class Batches(xgb.DataIter):
    def __init__(self, batches, fail_at=None):
        super().__init__(cache_prefix="unused", release_data=True, on_host=True)
        self.batches, self.i, self.calls, self.fail_at = batches, 0, [], fail_at

    def reset(self):
        self.calls.append("reset")
        self.i = 0

    def next(self, input_data):
        self.calls.append("next")
        if self.i == self.fail_at:
            raise KeyError("batch %d" % self.i)
        if self.i == len(self.batches):
            return False
        input_data(**self.batches[self.i])
        self.i += 1
        return True


def _batches():
    rng = np.random.default_rng(0)
    X = rng.standard_normal((10, 3)).astype(np.float32)
    y = np.arange(10, dtype=np.float32)
    qid = np.array([0, 0, 0, 1, 1, 1, 1, 2, 2, 2])              # the run of 1s crosses the batch boundary at row 5
    return X, y, qid, [dict(data=X[:5], label=y[:5], qid=qid[:5]), dict(data=X[5:].astype(np.float64), label=y[5:], qid=qid[5:])]


def test_call_order_and_batches(engine):
    X, y, qid, batches = _batches()
    it = Batches(batches)
    d = xgb.QuantileDMatrix(it, max_bin=64, missing=-1.0)
    assert d.handle == "qdm" and d.max_bin == 64 and engine.max_bin == 64 and engine.missing == -1.0
    assert it.calls == ["reset", "next", "next", "next"] * 2
    assert engine.freed == ["proxy"]
    for p in engine.passes:
        assert [x for x in p if isinstance(x, str)] == ["reset", "next", "next", "next"]
        got = [x for x in p if isinstance(x, dict)]
        assert [g["shape"] for g in got] == [(5, 3), (5, 3)]
        assert [g["dtype"] for g in got] == ["<f4", "<f8"]          # other dtypes go to the engine as they are, converted there
        np.testing.assert_array_equal(np.concatenate([g["label"] for g in got]), y)
        np.testing.assert_array_equal(np.concatenate([g["qid"] for g in got]), qid)
        assert all(g["label"].dtype == np.float32 for g in got)


def test_in_memory_data_is_one_batch(engine):
    import scipy.sparse as sp
    X, y, qid, _ = _batches()
    with pytest.warns(UserWarning, match="max_bin=1000"):
        xgb.QuantileDMatrix(sp.csr_matrix(X), label=y, group=[3, 4, 3], max_bin=1000)
    assert engine.max_bin == 256                                     # clamped, as the training parameter is
    (p1, p2) = engine.passes
    assert p1[:2] == ["reset", "next"] and p1[-1] == "next" and len(p1) == 4
    g = p1[2]
    assert g["kind"] == "csr" and g["rows"] == 10 and g["dtypes"] == ("<u8", "<u4", "<f4")
    np.testing.assert_array_equal(g["qid"], qid)                    # group sizes become the qid runs


def test_iterator_errors_are_reraised(engine):
    _, _, _, batches = _batches()
    with pytest.raises(KeyError):
        xgb.QuantileDMatrix(Batches(batches, fail_at=1))
    assert engine.freed[-1] == "qdm"


def test_meta_goes_through_input_data(engine):
    _, y, _, batches = _batches()
    with pytest.raises(xgb.XGBoostError, match="label"):
        xgb.QuantileDMatrix(Batches(batches), label=y)


def test_dmatrix_of_an_iterator_points_to_quantile_dmatrix():
    with pytest.raises(xgb.XGBoostError, match="QuantileDMatrix"):
        xgb.DMatrix(Batches([]))


def test_exported_names():
    assert xgb.QuantileDMatrix is core.QuantileDMatrix and xgb.DataIter is core.DataIter   # xgboost.core is this core module
    assert issubclass(core.QuantileDMatrix, core.DMatrix)
