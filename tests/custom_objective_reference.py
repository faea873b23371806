"""Custom-objective rounds restated on the CPU with the unchanged oracle trainer, and the oracle engine that runs the Python
layer on them (CPU tests of `Booster.update(fobj)`, `boost`, the sklearn decorator and `cv`).

`PairTrainer.boost(g, h)` grows one round's tree from caller-given pairs.  It runs the oracle's `reg:squarederror` trainer at
margin 0 on carrier labels c and weights h: that objective's pair is then (fl((0 - c) * h), h), so h is exact, and c is
picked among fl(-g / h) and its two float neighbours to give exactly g where one of them does (always when h is a power of
two, e.g. 1).  The trainer's subsample mask, fixed-point grid (`set_device_grid`) and growth apply to those pairs as to its
own.  This is the restatement tests/quantile_reference.py uses for the quantile pairs."""
import numpy as np

from oracle import gbt_oracle as O
from oracle.engine import OracleBackend

f32 = np.float32


def carrier(g, h):
    """Labels c with fl((0 - c) * h) == g wherever a float32 c does it; (g, h) with h == 0 needs g == 0."""
    g, h = np.asarray(g, f32), np.asarray(h, f32)
    if np.any((h == 0) & (g != 0)):
        raise ValueError("a pair with h == 0 and g != 0 has no carrier label")
    safe = np.where(h == 0, f32(1), h)
    c = (-(g / safe)).astype(f32)
    for d in (np.inf, -np.inf):
        miss = (-c * safe).astype(f32) != g
        if not miss.any():
            break
        alt = np.nextafter(c, f32(d)).astype(f32)
        c = np.where(miss & ((-alt * safe).astype(f32) == g), alt, c)
    return np.where(h == 0, f32(0), c).astype(f32)


class PairTrainer:
    """One output's trees grown from caller-given (g, h) pairs (the oracle's side of a custom round).  params: the booster's
    parameters (their objective sets the base margin and the exported model's objective)."""

    def __init__(self, params, X, base_score=0.5):
        self.params = dict(params)
        self.base_score = float(base_score)
        grow = {k: v for k, v in params.items() if k not in ("objective", "num_class", "scale_pos_weight", "base_score")}
        n = np.asarray(X).shape[0]
        self.t = O.Trainer(dict(grow, objective="reg:squarederror"), X=X, y=np.zeros(n, f32), weights=np.ones(n, f32), base_score=0.5)
        bm = O.base_margin_of({"objective": params.get("objective", "reg:squarederror"), "num_class": 1, "base_score": self.base_score})
        self.margin = np.full(n, bm, f32)
        self._zero = np.zeros(n, f32)

    @property
    def n(self):
        return self.t.n

    K = 1

    def set_device_grid(self, n=None):
        self.t.set_device_grid(n)

    def boost(self, g, h):
        g, h = np.asarray(g, f32).reshape(-1), np.asarray(h, f32).reshape(-1)
        self.t.y[:] = carrier(g, h)            # the trainer reads its label and weight arrays in place
        self.t.w[:] = h
        self.t.set_margins(self._zero)
        self.t.update()
        self.margin = (self.margin + self.t.margins()[:, 0]).astype(f32)

    def margins(self):
        return self.margin.reshape(-1, 1).copy()

    def update(self):
        raise ValueError("oracle engine: a round of the configured objective after custom rounds is not restated")

    def model(self):
        m = self.t.model()
        m["base_score"] = self.base_score
        m["objective"] = self.params.get("objective", "reg:squarederror")
        return m


class CustomObjectiveOracleBackend(OracleBackend):
    """The oracle engine with custom rounds through `PairTrainer` (one output).  It checks the pairs as the CUDA engine does
    (shape, finite values, h >= 0) and reads no labels."""

    def _pair_trainer(self, h, dh):
        if isinstance(h.trainer, PairTrainer) and h.trainer_dm is dh:
            return h.trainer
        if h.trainer is not None or h.loaded is not None:
            raise self.err("oracle engine: custom rounds are restated on a fresh booster and one training matrix only")
        if h.K() != 1:
            raise self.err("oracle engine: custom rounds are restated for one output")
        params = {k: (float(v) if isinstance(v, str) and k not in ("objective", "tree_method", "grow_policy", "booster") else v) for k, v in h.params.items()}
        params["objective"] = h.objective()
        for k in ("max_depth", "num_class", "max_bin", "seed", "max_leaves"):
            if k in params:
                params[k] = int(float(params[k]))
        h.trainer = PairTrainer(params, dh.X, float(params.get("base_score", 0.5)))
        h.trainer_dm = dh
        h.num_feature = dh.X.shape[1]
        return h.trainer

    def booster_training_margin(self, h, dh):
        return self._pair_trainer(h, dh).margins()

    def booster_boost(self, h, dh, it, grad, hess):
        t = self._pair_trainer(h, dh)
        n, K = t.n, t.K
        for what, a in (("grad", grad), ("hess", hess)):
            if not isinstance(a, np.ndarray):
                raise self.err("oracle engine: %s must be a numpy array" % what)
            if a.shape != (n, K):
                raise self.err("custom objective: %s has shape %s but the model trains (%d, %d) outputs on this matrix" % (what, a.shape, n, K))
        g, hs = grad.astype(f32), hess.astype(f32)
        bad = ~np.isfinite(g) | ~np.isfinite(hs) | (hs < 0)
        if bad.any():
            r, k = divmod(int(np.flatnonzero(bad.reshape(-1))[0]), K)
            raise self.err("custom objective: the gradient pair at row %d, output column %d is invalid" % (r, k))
        t.boost(g, hs)
