"""tests/ranking_reference.py against brute force and scikit-learn, the libsvm loaders on qid files, and the rejection of query
groups and rank:* objectives by an engine without them (the oracle's)."""
import numpy as np
import pytest

import ranking_reference as RR


def test_delta_ndcg_closed_form_matches_brute_force_swap():
    rng = np.random.default_rng(0)
    for trial in range(200):
        n = int(rng.integers(2, 30))
        y = rng.integers(0, 4, n).astype(np.float64)          # many ties
        exp_gain = bool(trial % 2)
        inv = RR.inv_idcg(y, n, exp_gain)
        base = RR.dcg(y, exp_gain)
        for a in range(n):
            for b in range(a + 1, n):
                z = y.copy()
                z[a], z[b] = z[b], z[a]
                want = abs(base - RR.dcg(z, exp_gain)) * inv
                assert RR.delta_ndcg(y, a, b, exp_gain, inv) == pytest.approx(want, rel=1e-12, abs=1e-15)


@pytest.mark.parametrize("R", ["zero", "one", "all", "random"])
def test_delta_map_closed_form_matches_brute_force_swap(R):
    rng = np.random.default_rng(1)
    for _ in range(100):
        n = int(rng.integers(1, 25))
        rel = {"zero": np.zeros(n), "one": np.eye(1, n, int(rng.integers(0, n)))[0], "all": np.ones(n),
               "random": (rng.random(n) < 0.4).astype(float)}[R]
        H, Q = RR.map_prefix(rel)
        ap = RR.average_precision(rel)
        pairs = 0
        for a in range(n):
            for b in range(a + 1, n):
                if rel[a] == rel[b]:
                    continue
                pairs += 1
                z = rel.copy()
                z[a], z[b] = z[b], z[a]
                want = abs(ap - RR.average_precision(z)) * rel.sum()
                assert RR.delta_map(H, Q, rel[a] > 0, a, b) == pytest.approx(want, rel=1e-12, abs=1e-14)
        if R in ("zero", "all"):
            assert pairs == 0


def _groups(rng, G, lo, hi):
    sizes = rng.integers(lo, hi + 1, G)
    return np.concatenate([[0], np.cumsum(sizes)])


def test_ndcg_metric_matches_sklearn():
    from sklearn.metrics import ndcg_score
    rng = np.random.default_rng(2)
    ptr = _groups(rng, 60, 2, 30)
    n = ptr[-1]
    y = rng.integers(0, 5, n).astype(np.float32)
    for g in range(60):                                          # at least one relevant document per group
        y[ptr[g]] = max(y[ptr[g]], 1)
    s = rng.permutation(n).astype(np.float32)                    # distinct scores
    for k in (None, 1, 3, 10):
        want = np.mean([ndcg_score(y[None, ptr[g]:ptr[g + 1]], s[None, ptr[g]:ptr[g + 1]], k=k) for g in range(60)])
        got = RR.metric(s, y, ptr, name="ndcg" if k is None else "ndcg@%d" % k, exp_gain=False)
        assert got == pytest.approx(want, rel=1e-12)


def test_map_metric_matches_sklearn():
    from sklearn.metrics import average_precision_score
    rng = np.random.default_rng(3)
    ptr = _groups(rng, 80, 2, 40)
    n = ptr[-1]
    y = (rng.random(n) < 0.3).astype(np.float32)
    for g in range(80):
        y[ptr[g]] = 1.0
    s = rng.permutation(n).astype(np.float32)
    want = np.mean([average_precision_score(y[ptr[g]:ptr[g + 1]], s[ptr[g]:ptr[g + 1]]) if y[ptr[g]:ptr[g + 1]].min() == 0 else 1.0
                    for g in range(80)])
    assert RR.metric(s, y, ptr, name="map") == pytest.approx(want, rel=1e-12)


def test_metric_groups_without_relevant_documents():
    y = np.zeros(4, np.float32)
    s = np.arange(4, dtype=np.float32)
    for name, v in (("ndcg", 1.0), ("ndcg-", 0.0), ("map", 1.0), ("map@2-", 0.0)):
        assert RR.metric(s, y, [0, 4], name=name) == v


def test_gradient_pair_rules():
    """Equal labels make no pair, pairs sum to zero in g, every h >= 0, and the topk pairs are those with a position < K."""
    rng = np.random.default_rng(4)
    ptr = _groups(rng, 40, 1, 50)
    n = ptr[-1]
    y = rng.integers(0, 3, n).astype(np.float32)
    m = rng.standard_normal(n).astype(np.float32)
    for obj in ("rank:pairwise", "rank:ndcg"):
        gp = RR.gradient(m, y, ptr, objective=obj, k=5, normalization=False)
        assert np.all(gp[:, 1] >= 0)
        for g in range(40):
            assert abs(gp[ptr[g]:ptr[g + 1], 0].astype(np.float64).sum()) < 1e-5
    same = RR.gradient(m, np.ones(n, np.float32), ptr, objective="rank:pairwise")
    assert np.all(same == 0)
    # K >= n: every pair; the order of evaluation does not change which pairs there are
    full = RR.gradient(m[:20], y[:20], [0, 20], objective="rank:pairwise", k=20, normalization=False, score_normalization=False)
    want = np.zeros(20)
    for i in range(20):
        for j in range(20):
            if y[i] > y[j]:
                sig = 1.0 / (1.0 + np.exp(-(float(m[i]) - float(m[j]))))
                want[i] += sig - 1.0
                want[j] -= sig - 1.0
    np.testing.assert_allclose(full[:, 0], want, rtol=1e-6, atol=1e-7)


def test_qid_to_group_ptr():
    np.testing.assert_array_equal(RR.group_ptr_from_qid([3, 3, 5, 5, 5, 9]), [0, 2, 5, 6])
    with pytest.raises(ValueError, match="non-decreasing"):
        RR.group_ptr_from_qid([1, 2, 1])


def _write_libsvm(tmp_path, rng, with_qid):
    files, qids = [], []
    q = 0
    for k in range(3):
        lines = []
        for r in range(int(rng.integers(1, 30))):
            if rng.random() < 0.3:
                q += int(rng.integers(1, 3))
            idx = np.sort(rng.choice(20, size=int(rng.integers(0, 6)), replace=False))
            toks = ["%d" % rng.integers(0, 4)] + (["qid:%d" % q] if with_qid else []) + ["%d:%.6g" % (i, v) for i, v in zip(idx, rng.standard_normal(len(idx)))]
            lines.append(" ".join(toks))
            qids.append(q)
        p = tmp_path / ("part-%d" % k)
        p.write_text("\n".join(lines) + "\n")
        files.append(str(p))
    return files, np.asarray(qids)


def test_libsvm_loaders_agree_on_qid_files(tmp_path):
    """A qid file goes to the plain loop (scikit-learn's parser would drop the tokens); its features and labels match the same
    file without the tokens through the fast parser, and the qid come back per row."""
    from sagemaker_xgboost_container_b200 import data
    (tmp_path / "q").mkdir()
    (tmp_path / "p").mkdir()
    files_q, qids = _write_libsvm(tmp_path / "q", np.random.default_rng(5), True)
    files_p, _ = _write_libsvm(tmp_path / "p", np.random.default_rng(5), False)
    assert data._load_libsvm_fast(files_q) is None
    Xq, yq, wq, q = data._load_libsvm(files_q, {}, with_qid=True)
    Xp, yp, wp = data._load_libsvm_fast(files_p)
    np.testing.assert_array_equal(q, qids)
    np.testing.assert_array_equal(yq, yp)
    assert wq is None and wp is None and Xq.shape[0] == Xp.shape[0] and (Xq[:, :Xp.shape[1]] != Xp).nnz == 0
    Xn, yn, wn, qn = data._load_libsvm(files_p, {}, with_qid=True)
    assert qn is None
    # a qid on a later line only still leaves the fast parser
    late = tmp_path / "late"
    late.write_text("1 0:1\n0 qid:4 1:2\n")
    assert data._load_libsvm_fast([str(late)]) is None
    with pytest.raises(Exception, match="all or none"):
        data._load_libsvm([str(late)], {}, with_qid=True)


def test_engine_without_ranking_rejects_groups_and_rank_objectives(monkeypatch):
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import backend
    from oracle.engine import OracleBackend
    monkeypatch.setattr(backend, "_BACKEND", OracleBackend(error_cls=xgb.XGBoostError))
    X = np.random.default_rng(6).standard_normal((10, 3)).astype(np.float32)
    with pytest.raises(xgb.XGBoostError, match="query groups .* not implemented by this engine"):
        xgb.DMatrix(X, label=np.zeros(10), group=[4, 6])
    with pytest.raises(xgb.XGBoostError, match="not implemented by this engine"):
        xgb.DMatrix(X, label=np.zeros(10), qid=np.repeat([1, 2], 5))
    d = xgb.DMatrix(X, label=np.zeros(10))
    with pytest.raises(xgb.XGBoostError, match="not implemented by this engine"):
        d.set_group([10])
    with pytest.raises(xgb.XGBoostError, match="not implemented by this engine"):
        xgb.train({"objective": "rank:ndcg"}, d, 1)
    assert len(d.get_group()) == 0
