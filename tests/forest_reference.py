"""Boosted random forests (num_parallel_tree = P > 1) restated on top of the oracle's Trainer (TEST INFRASTRUCTURE): the
per-tree row samples of csrc/booster.cu (update_one_iter), the fl(eta / P) leaves, the class-major layer layout and the
column streams keyed by the tree's position in the model.  Also an oracle engine that trains, indexes and writes forests.

Every tree of the model is grown by an oracle Trainer of its own, built so that its next tree is exactly that tree:
  * its sample weights are the tree's row sample (times the user's weights): unsampled rows get exactly (0, 0) (multi:softprob
    keeps a 1e-16 hessian there, below the fixed-point grid), and the fixed-point scale is max|g| / max h over the tree's
    sampled pairs of all K classes, as on the device;
  * its margins are set back to the round's starting margin, so all trees of a round fit the same gradients;
  * the oracle numbers the tree of class c in its update u as u * K + c.  Tree (round r, class k, j) sits at position
    t = indptr[r] + k * P + j of the model, so the Trainer is advanced to update u = t // K by throw-away updates, and class k is
    swapped with class c = t % K in the labels and margin columns.  The swap only reorders the softmax sum (last-bit changes);
    at K = 1, or whenever c == k, the tree is the product's to the bit."""
import numpy as np

from oracle import gbt_oracle as O
from oracle.engine import OracleBackend, _jsonable, _model_to_doc

from split_reference import rng_uniform

f32 = np.float32
FOREST_ROW_STREAM = 0x40000000000
KEYS = ("left", "right", "parent", "split_index", "split_bin", "default_left", "split_cond", "base_weight", "loss_chg", "sum_hess")


def row_stream(rnd, j):
    """The stream tree j of boosting round rnd draws its rows from: tree 0 keeps the single-tree stream."""
    return 0x2000 + rnd if j == 0 else FOREST_ROW_STREAM + (rnd << 20) + j


def row_mask(seed, rnd, j, n, subsample):
    if subsample >= 1.0:
        return np.ones(n, bool)
    return rng_uniform(seed, row_stream(rnd, j), np.arange(n, dtype=np.uint64)) < f32(subsample)


def forest_eta(eta, P):
    return f32(f32(eta) / f32(P))


def parse_num_parallel_tree(v):
    """The product's rule: an integer >= 1 written as a number or a string (no trailing characters)."""
    try:
        f = float(str(v).strip())
    except ValueError:
        raise ValueError("num_parallel_tree must be an integer in [1, 1048576] (got %r)" % (v,))
    if not (f == int(f) and 1 <= f <= (1 << 20)):
        raise ValueError("num_parallel_tree must be an integer in [1, 1048576] (got %r)" % (v,))
    return int(f)


def leaf_values(model, X, t):
    nid = O.predict_leaf(model, X, t, t + 1)[:, 0]
    return model["split_cond"][int(model["tree_offset"][t]) + nid].astype(np.float32)


def _tree_of(model, t):
    a, b = int(model["tree_offset"][t]), int(model["tree_offset"][t + 1])
    return {k: np.asarray(model[k][a:b]).copy() for k in KEYS}


class ForestTrainer:
    """One update() = one forest round of K * P trees; model() returns them in the product's class-major order."""

    def __init__(self, params, X, y, P, bins=None, cuts=None, base_score=None, weights=None, device_grid=True):
        self.P = int(P)
        self.params = dict(params)
        self.X = np.ascontiguousarray(X, np.float32)
        self.y = np.ascontiguousarray(y, np.float32)
        self.n = self.X.shape[0]
        self.sw = None if weights is None else np.ascontiguousarray(weights, np.float32)
        self.seed = int(params.get("seed", 0))
        self.subsample = float(params.get("subsample", 1.0))
        eta = float(params.get("eta", params.get("learning_rate", 0.3)))
        self.inner = dict(params, eta=float(forest_eta(eta, self.P)), subsample=1.0)
        self.inner.pop("learning_rate", None)
        if bins is None:
            cuts = O.make_cuts(self.X, int(params.get("max_bin", 256)), self.sw)
            bins = O.bin_matrix(self.X, cuts[0], cuts[1])
        self.bins, self.cuts = bins, cuts
        self.device_grid = device_grid
        self.K = max(1, int(params.get("num_class", 1) or 1)) if str(params.get("objective", "")).startswith("multi") else 1
        probe = self._trainer(np.ones(self.n, np.float32) if self.sw is None else self.sw, self.y, base_score)
        self.base_score = probe.base_score if base_score is None else float(base_score)
        self.m = probe.margins()
        self.trees, self.info, self.indptr = [], [], [0]

    def _trainer(self, w, y, base_score):
        t = O.Trainer(self.inner, y=y, weights=w, bins=self.bins, cuts=self.cuts, base_score=base_score)
        if self.device_grid:
            t.set_device_grid(self.n)
        return t

    def _grow(self, pre, pos, k, mask):
        K = self.K
        u, c = divmod(pos, K)
        perm = np.arange(K)
        perm[[k, c]] = perm[[c, k]]                       # product class -> oracle class
        y = perm[self.y.astype(np.int64)].astype(np.float32) if K > 1 else self.y
        w = mask.astype(np.float32) if self.sw is None else mask.astype(np.float32) * self.sw
        t = self._trainer(w, y, self.base_score)
        for _ in range(u):                                # throw-away updates: the next one is update u
            t.update()
        m = np.empty_like(pre)
        m[:, perm] = pre
        t.set_margins(m)
        t.update()
        model = t.model()
        assert int(model["tree_info"][u * K + c]) == c
        return _tree_of(model, u * K + c)

    def update(self):
        pre = self.m.copy()
        K, P, r = self.K, self.P, len(self.indptr) - 1
        masks = [row_mask(self.seed, r, j, self.n, self.subsample) for j in range(P)]
        for k in range(K):
            for j in range(P):
                tree = self._grow(pre, len(self.trees), k, masks[j])
                self.trees.append(tree)
                self.info.append(k)
                one = self.model(len(self.trees) - 1)
                self.m[:, k] = self.m[:, k] + leaf_values(one, self.X, 0)
        self.indptr.append(len(self.trees))

    def margins(self):
        return self.m.copy()

    def model(self, only=None):
        """The trees in model order as oracle.Model (only: just that tree)."""
        ids = range(len(self.trees)) if only is None else [only]
        out = O.Model()
        offs = [0]
        for k in KEYS:
            out[k] = np.concatenate([self.trees[t][k] for t in ids]) if len(ids) else np.zeros(0, np.float32 if k in
                                                                                                 ("split_cond", "base_weight", "loss_chg", "sum_hess") else np.int32)
        for t in ids:
            offs.append(offs[-1] + len(self.trees[t]["left"]))
        out["tree_offset"] = np.asarray(offs, np.int64)
        out["tree_info"] = np.asarray([self.info[t] for t in ids], np.int32)
        out["base_score"] = self.base_score
        out["num_class"] = self.K
        out["num_feature"] = self.X.shape[1]
        out["objective"] = self.params.get("objective", "reg:squarederror")
        return out


class ForestOracleBackend(OracleBackend):
    """The oracle engine with num_parallel_tree: trains forests with ForestTrainer, counts, predicts and slices by boosting round
    through the layer layout, and writes num_parallel_tree and iteration_indptr (CPU tests of the package's Python surface)."""

    def _P(self, h):
        try:
            P = parse_num_parallel_tree(h.params.get("num_parallel_tree", 1))
        except ValueError as e:
            raise self.err(str(e))
        if P > 1 and h.params.get("booster") == "dart":
            raise self.err("booster=dart with num_parallel_tree > 1 is not implemented")
        return P

    def _ensure_trainer(self, h, dh):
        P = self._P(h)
        if P == 1 and not isinstance(h.trainer, ForestTrainer):
            return super()._ensure_trainer(h, dh)
        if h.trainer is not None and h.trainer_dm is dh:
            return
        if h.trainer is not None or h.loaded is not None:
            raise self.err("oracle forest engine: training on a changed matrix or a loaded model is not restated")
        params = {k: (float(v) if isinstance(v, str) and k not in ("objective", "tree_method", "grow_policy", "booster") else v)
                  for k, v in h.params.items()}
        params["objective"] = h.objective()
        for k in ("max_depth", "num_class", "max_bin", "seed", "max_leaves"):
            if k in params:
                params[k] = int(float(params[k]))
        y = dh.info["label"]
        w = dh.info["weight"] if len(dh.info["weight"]) else None
        h.trainer = ForestTrainer(params, dh.X, y, P, weights=w, device_grid=False)
        h.trainer_dm = dh
        h.num_feature = dh.X.shape[1]

    def _indptr(self, h):
        if isinstance(h.trainer, ForestTrainer):
            return list(h.trainer.indptr)
        if getattr(h, "forest_indptr", None) is not None:
            return list(h.forest_indptr)
        K, nt = h.K(), len(h.model()["tree_info"])
        return list(range(0, nt + 1, K))

    def booster_boosted_rounds(self, h):
        return len(self._indptr(h)) - 1

    def booster_predict(self, h, dh, cfg):
        ip = self._indptr(h)
        b, e = int(cfg.get("iteration_begin", 0)), int(cfg.get("iteration_end", 0))
        e = len(ip) - 1 if e == 0 else e
        if not 0 <= b <= e <= len(ip) - 1:
            raise self.err("Invalid iteration range: [%d, %d)" % (b, e))
        m = h.model()
        n = dh.X.shape[0]
        if cfg.get("type", 0) == 6:
            return O.predict_leaf(m, dh.X, ip[b], ip[e]).astype(np.float32)
        _, margin = self._margin(h, dh, ip[b], ip[e])
        out = np.asarray(margin if cfg.get("type", 0) == 1 else O.transform(m, margin), np.float32)
        if out.ndim == 2 and out.shape[1] == 1 and not cfg.get("strict_shape"):
            out = out[:, 0]
        elif out.ndim == 1 and cfg.get("strict_shape"):
            out = out.reshape(n, 1)
        return out

    def booster_slice(self, h, begin, end, step):
        ip = self._indptr(h)
        end = len(ip) - 1 if end == 0 else end
        if not (0 <= begin < end <= len(ip) - 1) or step < 1:
            raise self.err("Layer index out of range")
        m = h.model()
        keep = [t for r in range(begin, end, step) for t in range(ip[r], ip[r + 1])]
        out = super().booster_slice(h, 0, 0, 1)              # copies the parameters; its trees are replaced below
        mm = O.Model()
        offs = [0]
        for k in KEYS:
            mm[k] = np.concatenate([m[k][int(m["tree_offset"][t]):int(m["tree_offset"][t + 1])] for t in keep])
        for t in keep:
            offs.append(offs[-1] + int(m["tree_offset"][t + 1] - m["tree_offset"][t]))
        mm["tree_offset"] = np.asarray(offs, np.int64)
        mm["tree_info"] = np.asarray(m["tree_info"][keep], np.int32)
        for k in ("base_score", "num_class", "num_feature", "objective"):
            mm[k] = m[k]
        out.loaded = mm
        new_ip = [0]
        for r in range(begin, end, step):
            new_ip.append(new_ip[-1] + ip[r + 1] - ip[r])
        out.forest_indptr = new_ip
        return out

    def _doc(self, h):
        doc = _model_to_doc(h.model(), h.attrs, h.names)
        model = doc["learner"]["gradient_booster"]["model"]
        model["gbtree_model_param"]["num_parallel_tree"] = str(self._P(h))
        model["iteration_indptr"] = np.asarray(self._indptr(h), np.int32)
        return doc

    def booster_save_raw(self, h, fmt):
        import json
        from oracle import ubjson
        doc = self._doc(h)
        return json.dumps(_jsonable(doc)).encode() if fmt == "json" else ubjson.dumps(doc)

    def booster_serialize(self, h):
        import json
        from oracle import ubjson
        return ubjson.dumps({"Model": self._doc(h), "Config": json.loads(self.booster_save_config(h))})

    def booster_save_config(self, h):
        import json
        cfg = json.loads(super().booster_save_config(h))
        cfg["learner"]["gradient_booster"]["gbtree_model_param"] = {"num_parallel_tree": str(self._P(h))}
        return json.dumps(cfg)

    def booster_load_raw(self, h, buf):
        import json
        from oracle import ubjson
        super().booster_load_raw(h, buf)
        raw = bytes(buf)
        try:
            doc = json.loads(raw.decode()) if raw[:2] in (b'{"', b"{ ", b"{\n") else ubjson.loads(raw)
        except Exception:
            return                                             # legacy binary formats are single-tree rounds
        model = doc.get("Model", doc)["learner"]["gradient_booster"]["model"]
        P = parse_num_parallel_tree(model.get("gbtree_model_param", {}).get("num_parallel_tree", 1))
        h.params["num_parallel_tree"] = str(P)
        ip = model.get("iteration_indptr")
        h.forest_indptr = [int(v) for v in ip] if ip is not None else list(range(0, len(model["tree_info"]) + 1, h.K() * P))
