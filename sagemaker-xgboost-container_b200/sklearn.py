"""scikit-learn style wrappers (`XGBRegressor`, `XGBClassifier`, `XGBRanker`) over `train()` -- the subset of `xgboost.sklearn` that
script-mode customer code in the container's test resources uses (test/resources/boston/single_machine_customer_script.py:54).
"""
import json

import numpy as np

from .core import Booster, DMatrix, XGBoostError
from .training import train

_FIT_ONLY = {"n_estimators", "early_stopping_rounds", "eval_metric", "callbacks", "missing", "importance_type", "enable_categorical",
             "feature_types", "n_jobs", "random_state", "verbosity", "objective", "kwargs"}


class XGBModel:
    _default_objective = "reg:squarederror"

    def __init__(self, max_depth=None, max_leaves=None, max_bin=None, grow_policy=None, learning_rate=None, n_estimators=None, verbosity=None,
                 objective=None, booster=None, tree_method=None, n_jobs=None, gamma=None, min_child_weight=None, max_delta_step=None,
                 subsample=None, colsample_bytree=None, colsample_bylevel=None, colsample_bynode=None, reg_alpha=None, reg_lambda=None,
                 scale_pos_weight=None, base_score=None, random_state=None, missing=np.nan, importance_type=None, device=None,
                 early_stopping_rounds=None, eval_metric=None, callbacks=None, **kwargs):
        for k, v in list(locals().items()):
            if k not in ("self", "kwargs", "__class__"):
                setattr(self, k, v)
        self.kwargs = kwargs
        self._Booster = None
        self.evals_result_ = {}

    # ---- sklearn plumbing
    def get_params(self, deep=True):
        code = XGBModel.__init__.__code__
        p = {k: getattr(self, k) for k in code.co_varnames[1:code.co_argcount]}
        p.update(self.kwargs)
        return p

    def set_params(self, **params):
        for k, v in params.items():
            if hasattr(self, k):
                setattr(self, k, v)
            else:
                self.kwargs[k] = v
        return self

    def get_xgb_params(self):
        p = {k: v for k, v in self.get_params().items() if v is not None and k not in _FIT_ONLY}
        p["objective"] = self.objective or self._default_objective
        if self.random_state is not None:
            p["seed"] = int(self.random_state)
        if self.eval_metric is not None and not callable(self.eval_metric):
            p["eval_metric"] = self.eval_metric
        p.pop("device", None)
        return p

    def get_num_boosting_rounds(self):
        return 100 if self.n_estimators is None else int(self.n_estimators)

    def get_booster(self):
        if self._Booster is None:
            raise XGBoostError("need to call fit or load_model beforehand")
        return self._Booster

    def _dmatrix(self, X, y=None, sample_weight=None, base_margin=None):
        return DMatrix(X, label=y, weight=sample_weight, base_margin=base_margin, missing=self.missing)

    def _fit(self, params, X, y, sample_weight, base_margin, eval_set, sample_weight_eval_set, verbose, xgb_model):
        dtrain = self._dmatrix(X, y, sample_weight, base_margin)
        evals = []
        for i, (Xe, ye) in enumerate(eval_set or []):
            we = sample_weight_eval_set[i] if sample_weight_eval_set else None
            evals.append((dtrain if (Xe is X and ye is y) else self._dmatrix(Xe, ye, we), "validation_%d" % i))
        self.evals_result_ = {}
        model = xgb_model.get_booster() if isinstance(xgb_model, XGBModel) else xgb_model
        self._Booster = train(params, dtrain, self.get_num_boosting_rounds(), evals=evals, early_stopping_rounds=self.early_stopping_rounds,
                              evals_result=self.evals_result_, custom_metric=self.eval_metric if callable(self.eval_metric) else None,
                              verbose_eval=verbose, xgb_model=model, callbacks=self.callbacks)
        self.n_features_in_ = dtrain.num_col()
        return self

    def fit(self, X, y, *, sample_weight=None, base_margin=None, eval_set=None, verbose=True, xgb_model=None, sample_weight_eval_set=None):
        return self._fit(self.get_xgb_params(), X, y, sample_weight, base_margin, eval_set, sample_weight_eval_set, verbose, xgb_model)

    def _iteration_range(self, iteration_range):
        if iteration_range is None or iteration_range[1] == 0:
            try:
                return (0, self.get_booster().best_iteration + 1)
            except AttributeError:
                return (0, 0)
        return iteration_range

    def predict(self, X, output_margin=False, validate_features=True, base_margin=None, iteration_range=None):
        d = self._dmatrix(X, base_margin=base_margin)
        return self.get_booster().predict(d, output_margin=output_margin, validate_features=validate_features,
                                          iteration_range=self._iteration_range(iteration_range))

    def apply(self, X, iteration_range=None):
        return self.get_booster().predict(self._dmatrix(X), pred_leaf=True, iteration_range=self._iteration_range(iteration_range))

    def evals_result(self):
        return self.evals_result_

    @property
    def best_iteration(self):
        return self.get_booster().best_iteration

    @property
    def best_score(self):
        return self.get_booster().best_score

    @property
    def feature_importances_(self):
        b = self.get_booster()
        score = b.get_score(importance_type=self.importance_type or "gain")
        names = b.feature_names or ["f%d" % i for i in range(b.num_features())]
        arr = np.array([score.get(n, 0.0) for n in names], dtype=np.float32)
        tot = arr.sum()
        return arr / tot if tot > 0 else arr

    def save_model(self, fname):
        self.get_booster().save_model(fname)

    def load_model(self, fname):
        self._Booster = Booster(model_file=fname)
        cfg = json.loads(self._Booster.save_config())
        self.objective = cfg["learner"]["objective"]["name"]
        self.n_features_in_ = self._Booster.num_features()


class XGBRegressor(XGBModel):
    _default_objective = "reg:squarederror"


class XGBClassifier(XGBModel):
    _default_objective = "binary:logistic"

    def fit(self, X, y, *, sample_weight=None, base_margin=None, eval_set=None, verbose=True, xgb_model=None, sample_weight_eval_set=None):
        y = np.asarray(y)
        if y.ndim == 2 and y.shape[1] > 1:
            # multi-label classification is not implemented: the label reaches the engine flat, which refuses its n * T entries
            # ("labels are not correctly provided") rather than training T binary:logistic targets
            y = y.reshape(-1)
        self.classes_ = np.unique(y)
        self.n_classes_ = len(self.classes_)
        if not np.array_equal(self.classes_, np.arange(self.n_classes_)):
            raise ValueError("Invalid classes inferred from unique values of `y`.  Expected: %s, got %s" % (np.arange(self.n_classes_), self.classes_))
        params = self.get_xgb_params()
        if self.n_classes_ > 2:
            if not str(params["objective"]).startswith("multi:"):
                params["objective"] = "multi:softprob"
            params["num_class"] = self.n_classes_
        return self._fit(params, X, y, sample_weight, base_margin, eval_set, sample_weight_eval_set, verbose, xgb_model)

    def predict_proba(self, X, validate_features=True, base_margin=None, iteration_range=None):
        p = XGBModel.predict(self, X, validate_features=validate_features, base_margin=base_margin, iteration_range=iteration_range)
        if p.ndim == 1:
            return np.vstack([1.0 - p, p]).T
        return p

    def predict(self, X, output_margin=False, validate_features=True, base_margin=None, iteration_range=None):
        if output_margin:
            return XGBModel.predict(self, X, True, validate_features, base_margin, iteration_range)
        p = self.predict_proba(X, validate_features, base_margin, iteration_range)
        return np.argmax(p, axis=1)


class XGBRanker(XGBModel):
    """Learning to rank over query groups: the rows of each query are given by `group` (sizes) or `qid` (one id per row, sorted),
    `sample_weight` holds one weight per group, and `predict` returns the ranking scores (margins)."""
    _default_objective = "rank:ndcg"

    def _ranking_dmatrix(self, X, y, group, qid, sample_weight=None, base_margin=None):
        if (group is None) == (qid is None):
            raise ValueError("XGBRanker needs exactly one of group and qid for every matrix it trains or evaluates on")
        return DMatrix(X, label=y, weight=sample_weight, base_margin=base_margin, missing=self.missing, group=group, qid=qid)

    def fit(self, X, y, *, group=None, qid=None, sample_weight=None, base_margin=None, eval_set=None, eval_group=None, eval_qid=None,
            verbose=False, xgb_model=None, sample_weight_eval_set=None):
        params = self.get_xgb_params()
        if not str(params["objective"]).startswith("rank:"):
            raise ValueError("XGBRanker takes a rank:* objective (got %s)" % params["objective"])
        dtrain = self._ranking_dmatrix(X, y, group, qid, sample_weight, base_margin)
        evals = []
        for i, (Xe, ye) in enumerate(eval_set or []):
            ge = eval_group[i] if eval_group is not None else None
            qe = eval_qid[i] if eval_qid is not None else None
            we = sample_weight_eval_set[i] if sample_weight_eval_set else None
            evals.append((self._ranking_dmatrix(Xe, ye, ge, qe, we), "validation_%d" % i))
        self.evals_result_ = {}
        model = xgb_model.get_booster() if isinstance(xgb_model, XGBModel) else xgb_model
        self._Booster = train(params, dtrain, self.get_num_boosting_rounds(), evals=evals, early_stopping_rounds=self.early_stopping_rounds,
                              evals_result=self.evals_result_, custom_metric=self.eval_metric if callable(self.eval_metric) else None,
                              verbose_eval=verbose, xgb_model=model, callbacks=self.callbacks)
        self.n_features_in_ = dtrain.num_col()
        return self

    def predict(self, X, output_margin=False, validate_features=True, base_margin=None, iteration_range=None):
        return XGBModel.predict(self, X, True, validate_features, base_margin, iteration_range)


class _RandomForest:
    """Random forests the way `xgboost.sklearn` builds them: one boosting round of `n_estimators` parallel trees
    (num_parallel_tree), each on its own row and column sample, with learning rate 1 and almost no L2 penalty."""

    def __init__(self, *, learning_rate=1.0, subsample=0.8, colsample_bynode=0.8, reg_lambda=1e-5, **kwargs):
        super().__init__(learning_rate=learning_rate, subsample=subsample, colsample_bynode=colsample_bynode, reg_lambda=reg_lambda, **kwargs)

    def get_xgb_params(self):
        p = super().get_xgb_params()
        p["num_parallel_tree"] = super().get_num_boosting_rounds()
        return p

    def get_num_boosting_rounds(self):
        return 1

    def _fit(self, *args, **kwargs):
        if self.early_stopping_rounds is not None or self.callbacks:
            raise NotImplementedError("`early_stopping_rounds` and `callbacks` are not implemented for random forest.")
        return super()._fit(*args, **kwargs)


class XGBRFRegressor(_RandomForest, XGBRegressor):
    pass


class XGBRFClassifier(_RandomForest, XGBClassifier):
    pass
