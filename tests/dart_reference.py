"""booster=dart restated on top of the oracle's Trainer (TEST INFRASTRUCTURE): the drop draws, the tree weights and the defined
margin arithmetic of csrc/booster.cu (dart_drop_set, dart_begin_round) and csrc/dart.cu, so that the product can be checked
against it bit for bit.  Also the weighted margin and Shapley values of a dart model, and an oracle engine that trains dart."""
import numpy as np

from oracle import gbt_oracle as O
from oracle.engine import OracleBackend
from split_reference import rng_uniform

f32 = np.float32
SKIP_STREAM, ONE_STREAM, TREE_STREAM = 0x10000000000, 0x20000000000, 0x30000000000


def dart_param(params):
    g = params.get
    return dict(rate_drop=float(g("rate_drop", 0.0)), skip_drop=float(g("skip_drop", 0.0)), one_drop=int(float(g("one_drop", 0))),
                sample_type=str(g("sample_type", "uniform")), normalize_type=str(g("normalize_type", "tree")))


def drop_set(weights, rnd, seed, dp):
    """The trees dropped in boosting round `rnd`, given the weights of the trees so far (every class)."""
    T = len(weights)
    if T == 0:
        return []
    if dp["skip_drop"] > 0 and rng_uniform(seed, SKIP_STREAM, rnd) < f32(dp["skip_drop"]):
        return []
    w = np.asarray(weights, np.float32)
    u = rng_uniform(seed, TREE_STREAM + rnd, np.arange(T, dtype=np.uint64))
    if dp["sample_type"] == "weighted":
        sum_w = f32(0)
        for x in w:
            sum_w = f32(sum_w + x)
        thr = [f32(f32(f32(f32(dp["rate_drop"]) * f32(T)) * w[i]) / sum_w) for i in range(T)]
    else:
        thr = [f32(dp["rate_drop"])] * T
    D = [i for i in range(T) if u[i] < thr[i]]
    if dp["one_drop"] and not D:
        uu = float(rng_uniform(seed, ONE_STREAM, rnd))
        pick = min(T - 1, int(uu * T))
        if dp["sample_type"] == "weighted":
            target, acc, pick = uu * float(np.sum(w.astype(np.float64))), 0.0, T - 1
            for i in range(T):
                acc += float(w[i])
                if acc > target:
                    pick = i
                    break
        D = [pick]
    return D


def normalisation(n_drop, eta, K, normalize_type):
    """(factor of the dropped trees' weights, weight of the new trees), in the float / double steps of dart_begin_round."""
    lr = f32(float(eta) / K)
    if n_drop == 0:
        return f32(1), f32(1)
    if normalize_type == "forest":
        factor = f32(1.0 / (1.0 + float(lr)))
        return factor, factor
    denom = f32(f32(n_drop) + lr)
    return f32(n_drop / float(denom)), f32(1.0 / float(denom))


def leaf_values(model, X, t):
    """Leaf value of tree t on every row (the oracle's traversal of the raw features)."""
    nid = O.predict_leaf(model, X, t, t + 1)[:, 0]
    return model["split_cond"][int(model["tree_offset"][t]) + nid].astype(np.float32)


class DartTrainer:
    """One `update()` = one dart round: margins without the drop set for the gradients, new weights, the defined cache update."""

    def __init__(self, params, X, y=None, weights=None, trainer=None):
        """trainer: an O.Trainer set up by the caller (e.g. on the device's bins and fixed-point grid); else one on X, y."""
        self.params = dict(params)
        self.dp = dart_param(params)
        self.X = np.ascontiguousarray(X, np.float32)
        self.t = trainer if trainer is not None else O.Trainer(params, X=self.X, y=y, weights=weights)
        self.K = self.t.K
        self.eta = float(params.get("eta", params.get("learning_rate", 0.3)))
        self.seed = int(params.get("seed", 0))
        self.weights = []
        self.drops = []
        self.m_full = None

    def model(self):
        return self.t.model()

    def update(self):
        T = len(self.weights)
        rnd = T // self.K
        D = drop_set(self.weights, rnd, self.seed, self.dp)
        self.drops.append(D)
        factor, w_new = normalisation(len(D), self.eta, self.K, self.dp["normalize_type"])
        if T:
            model = self.t.model()
            info = model["tree_info"]
            m_drop = self.m_full.copy()
            for j in D:                          # ascending: m_drop -= fl(w * leaf), m_full += fl(c * leaf), c = fl(w' - w)
                v = leaf_values(model, self.X, j)
                w = f32(self.weights[j])
                w2 = f32(w * factor)
                c = int(info[j])
                m_drop[:, c] = m_drop[:, c] - w * v
                self.m_full[:, c] = self.m_full[:, c] + f32(w2 - w) * v
                self.weights[j] = w2
            self.t.set_margins(m_drop)
        self.t.update()
        model = self.t.model()
        if T == 0:
            self.m_full = self.t.margins()       # base margin + fl(1 * leaf): the trainer's own sum
        else:
            for t in range(T, T + self.K):
                c = int(model["tree_info"][t])
                self.m_full[:, c] = self.m_full[:, c] + w_new * leaf_values(model, self.X, t)
        self.weights += [w_new] * self.K
        return D


def predict_margin(model, X, weights, tree_begin=0, tree_end=None, base_margin=None):
    """base + sum_t fl(w_t * leaf_t), added in tree order in float32."""
    X = np.ascontiguousarray(X, np.float32)
    K = int(model.get("num_class", 1))
    tree_end = len(model["tree_info"]) if tree_end is None else tree_end
    bm = O.base_margin_of(model) if base_margin is None else base_margin
    out = np.full((X.shape[0], K), bm, np.float32)
    for t in range(tree_begin, tree_end):
        c = int(model["tree_info"][t])
        out[:, c] = out[:, c] + f32(weights[t]) * leaf_values(model, X, t)
    return out


def shap_weighted(model, X, weights, tree_begin=0, tree_end=None):
    """Shapley values of sum_t w_t * tree_t (+ the base margin in the bias column), float64 (n, K, F + 1)."""
    tree_end = len(model["tree_info"]) if tree_end is None else tree_end
    base = O.shap_bruteforce(model, X, 0, 0)
    out = base.copy()
    for t in range(tree_begin, tree_end):
        out += float(weights[t]) * (O.shap_bruteforce(model, X, t, t + 1) - base)
    return out


class DartOracleBackend(OracleBackend):
    """The oracle engine with booster=dart: trains with DartTrainer and predicts the weighted margin (CPU tests of the container
    route).  Models it writes carry the dart document's weight_drop."""

    def _ensure_trainer(self, h, dh):
        if h.params.get("booster") != "dart":
            return super()._ensure_trainer(h, dh)
        if h.trainer is not None and h.trainer_dm is dh:
            return
        dp = dart_param(h.params)
        if dp["sample_type"] not in ("uniform", "weighted") or dp["normalize_type"] not in ("tree", "forest") or not (0 <= dp["rate_drop"] <= 1) \
                or not (0 <= dp["skip_drop"] <= 1) or dp["one_drop"] not in (0, 1):
            raise self.err("invalid DART parameters: %r" % (dp,))
        params = {k: v for k, v in h.params.items() if k not in ("sample_type", "normalize_type", "booster")}
        params = {k: (float(v) if isinstance(v, str) and k not in ("objective", "tree_method", "grow_policy") else v) for k, v in params.items()}
        params["objective"] = h.objective()
        for k in ("max_depth", "num_class", "max_bin", "seed", "max_leaves"):
            if k in params:
                params[k] = int(float(params[k]))
        params.update(sample_type=dp["sample_type"], normalize_type=dp["normalize_type"])
        w = dh.info["weight"] if len(dh.info["weight"]) else None
        h.trainer = DartTrainer(params, dh.X, dh.info["label"], weights=w)
        h.trainer_dm = dh
        h.num_feature = dh.X.shape[1]

    @staticmethod
    def _tree_weights(h):
        if isinstance(h.trainer, DartTrainer):
            return h.trainer.weights
        return getattr(h, "dart_weights", None)

    def _margin(self, h, dh, tree_begin=0, tree_end=None):
        w = self._tree_weights(h)
        if w is None:
            return super()._margin(h, dh, tree_begin, tree_end)
        m = h.model()
        return m, predict_margin(m, dh.X, w, tree_begin, tree_end)

    def _doc(self, h):
        from oracle.engine import _model_to_doc
        doc = _model_to_doc(h.model(), h.attrs, h.names)
        w = self._tree_weights(h)
        if w is not None:
            gb = doc["learner"]["gradient_booster"]
            doc["learner"]["gradient_booster"] = {"name": "dart", "gbtree": gb, "weight_drop": np.asarray(w, np.float32)}
        return doc

    def booster_save_raw(self, h, fmt):
        import json
        from oracle import ubjson
        from oracle.engine import _jsonable
        doc = self._doc(h)
        return json.dumps(_jsonable(doc)).encode() if fmt == "json" else ubjson.dumps(doc)

    def booster_serialize(self, h):
        import json
        from oracle import ubjson
        return ubjson.dumps({"Model": self._doc(h), "Config": json.loads(self.booster_save_config(h))})

    def booster_load_raw(self, h, buf):
        import json
        from oracle import ubjson
        buf = bytes(buf)
        doc = json.loads(buf.decode()) if buf[:2] in (b'{"', b"{ ", b"{\n") else ubjson.loads(buf)
        doc = doc.get("Model", doc)
        gb = doc["learner"]["gradient_booster"]
        if gb.get("name") != "dart":
            h.dart_weights = None
            return super().booster_load_raw(h, buf)
        doc["learner"]["gradient_booster"] = gb["gbtree"]
        super().booster_load_raw(h, ubjson.dumps(doc))
        h.dart_weights = [f32(v) for v in gb["weight_drop"]]
        h.params["booster"] = "dart"
