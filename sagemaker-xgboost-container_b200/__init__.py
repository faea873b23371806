"""H100-native (sm_90a) gradient-boosted trees behind the `xgboost` API surface used by aws/sagemaker-xgboost-container.

Import as a package (`import sagemaker_xgboost_container_b200 as xgb`, see the loader module at the repo root) or
bind it under the name `xgboost` with `install_as_xgboost()` so that the container's modules
(`sagemaker_xgboost_container.algorithm_mode.train`, `data_utils`, `checkpointing`, `distributed`, `serving`)
run unchanged on top of the CUDA engine (INTEGRATION.md).
"""
import sys

from . import callback, collective, core, dask, sklearn, tracker, training  # noqa: F401
from .backend import XGBoostError, get_backend  # noqa: F401
from .core import Booster, DataIter, DMatrix, QuantileDMatrix  # noqa: F401
from .training import cv, train  # noqa: F401
from .sklearn import XGBClassifier, XGBModel, XGBRanker, XGBRegressor, XGBRFClassifier, XGBRFRegressor  # noqa: F401

__version__ = "3.0.5"        # API level mirrored (docker/3.0-5/base/Dockerfile.cpu:33 pins xgboost==3.0.5)


def build_info():
    return get_backend().build_info()


def install_as_xgboost():
    """Alias this package as `xgboost` (+ the submodules the container imports) in sys.modules."""
    me = sys.modules[__name__]
    sys.modules["xgboost"] = me
    for sub in ("core", "callback", "collective", "tracker", "training", "sklearn", "dask"):
        sys.modules["xgboost." + sub] = getattr(me, sub)
    return me
