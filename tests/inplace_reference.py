"""The oracle engine with in-place prediction: it applies the engine's checks (2-D, dtype, feature count, predict type,
base_margin size) and then predicts on the matrix the DMatrix path builds from the same values converted to float32.  Lets
the CPU tests run the Python layer of `Booster.inplace_predict` (input kinds, conversions, shapes and errors)."""
import numpy as np

from oracle.engine import OracleBackend


class InplaceOracleBackend(OracleBackend):
    def _inplace(self, h, dm, cfg, base_margin):
        if cfg.get("type", 0) not in (0, 1):
            raise self.err("inplace_predict: predict type %s is not supported (0 value, 1 margin)" % cfg.get("type"))
        if h.num_feature and dm.X.shape[1] > h.num_feature:
            raise self.err("feature count mismatch: the data has %d columns, the model was trained on %d features" % (dm.X.shape[1], h.num_feature))
        if base_margin is not None:
            if len(base_margin) != dm.X.shape[0] * h.K():
                raise self.err("base_margin size does not match rows x groups")
            dm.info["base_margin"] = np.asarray(base_margin, np.float32).reshape(-1)
        return self.booster_predict(h, dm, cfg)

    def booster_inplace_dense(self, h, arr, cfg, base_margin=None):
        if arr.ndim != 2:
            raise self.err("inplace_predict: expecting a 2-dimensional array, got %d dimension(s)" % arr.ndim)
        dt = arr.dtype
        if dt.kind not in "fiub" or dt.byteorder == ">" or dt.itemsize > 8 or (dt.kind == "f" and dt.itemsize < 2):
            raise self.err("inplace_predict: unsupported typestr " + dt.str)
        return self._inplace(h, self.dmatrix_from_dense(arr.astype(np.float32), cfg.get("missing", np.nan)), cfg, base_margin)

    def booster_inplace_csr(self, h, indptr, indices, data, ncol, cfg, base_margin=None):
        if len(indices) and (int(np.min(indices)) < 0 or int(np.max(indices)) >= ncol):
            raise self.err("inplace_predict: CSR column index outside [0, %d)" % ncol)
        dm = self.dmatrix_from_csr(np.asarray(indptr), np.asarray(indices), np.asarray(data, np.float32), ncol)
        return self._inplace(h, dm, cfg, base_margin)
