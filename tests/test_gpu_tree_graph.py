"""Graph replay of the per-tree launch sequence equals issuing it directly (run with `pytest -m gpu` on an H100).

Every case trains twice, in two processes: once by default (trees replayed from captured CUDA graphs) and once with
B200XGB_NO_GRAPH=1 (every launch issued directly).  Every exported model array and every cached margin must agree bit for
bit.  The cases change what a captured graph depends on between rounds: parameters, the training matrix, constraints.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_TRAIN = r"""
import json, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import sagemaker_xgboost_container_b200 as xgb
from util import synth
cfg = json.loads(sys.argv[2])
mats = []
for n, F, seed, kind, K in cfg["data"]:
    X, y = synth(n, F, seed, kind, K=K, quantised=False)
    mats.append(xgb.DMatrix(X, label=y))
bst = xgb.Booster(cfg["params"], mats)
schedule = cfg.get("schedule") or []
for i in range(cfg["rounds"]):
    if i < len(schedule):
        bst.set_param(schedule[i])
    bst.update(mats[i % len(mats)], i)
be = xgb.get_backend()
out = {k: np.asarray(v) for k, v in be.booster_export_model(bst.handle).items()}
K = max(1, int(cfg["params"].get("num_class", 1)))
for j, d in enumerate(mats):
    out["cached_margin_%d" % j] = be.booster_cached_margin(bst.handle, d.handle, K)
np.savez(sys.argv[3], **out)
"""


def _train_in_subprocess(tmp_path, cfg, no_graph):
    env = dict(os.environ)
    env.pop("B200XGB_NO_GRAPH", None)
    if no_graph:
        env["B200XGB_NO_GRAPH"] = "1"           # read once per process: the two models are trained in two processes
    out = str(tmp_path / ("model_%d.npz" % no_graph))
    r = subprocess.run([sys.executable, "-s", "-c", _TRAIN, ROOT, json.dumps(cfg), out], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return dict(np.load(out))


_BASE = dict(tree_method="hist", max_bin=256, eta=0.3, max_depth=6)
_REG = [60000, 40, 3, "reg", 1]

CASES = {
    # constant hessian: the first tree takes root mode 1 (issued directly), the later ones mode 2 (replayed)
    "squarederror_depth6": dict(params=dict(_BASE, objective="reg:squarederror"), rounds=5, data=[_REG]),
    "logistic_100_features": dict(params=dict(_BASE, objective="binary:logistic"), rounds=5, data=[[60000, 100, 5, "bin", 1]]),
    "softprob_3_classes": dict(params=dict(_BASE, objective="multi:softprob", num_class=3), rounds=4, data=[[50000, 30, 7, "multi", 3]]),
    "lossguide_24_leaves": dict(params=dict(_BASE, objective="reg:squarederror", grow_policy="lossguide", max_leaves=24), rounds=5, data=[_REG]),
    "colsample_level_node": dict(params=dict(_BASE, objective="reg:squarederror", colsample_bylevel=0.5, colsample_bynode=0.5, seed=3),
                                 rounds=5, data=[_REG]),
    "monotone_interaction": dict(params=dict(_BASE, objective="reg:squarederror", monotone_constraints="(1,-1,0,1)",
                                             interaction_constraints="[[0, 1], [2, 3, 4], [5, 6, 7, 8]]"), rounds=5, data=[[60000, 12, 9, "reg", 1]]),
    # one parameter changes before every update; each is baked into a captured graph
    "set_param_every_round": dict(params=dict(_BASE, objective="binary:logistic"), rounds=11, data=[[60000, 40, 11, "bin", 1]],
                                  schedule=[{}, {"eta": "0.1"}, {"lambda": "3"}, {"alpha": "0.5"}, {"gamma": "0.2"}, {"min_child_weight": "20"},
                                            {"max_delta_step": "0.3"}, {"max_depth": "4"}, {"max_leaves": "9"}, {"colsample_bynode": "0.5"},
                                            {"seed": "17"}]),
    # one Booster updated alternately on two matrices with different row counts
    "two_matrices": dict(params=dict(_BASE, objective="reg:squarederror"), rounds=6, data=[_REG, [35000, 40, 13, "reg", 1]]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_graph_replay_equals_direct_issue(tmp_path, case):
    cfg = CASES[case]
    replayed = _train_in_subprocess(tmp_path, cfg, False)
    direct = _train_in_subprocess(tmp_path, cfg, True)
    assert (replayed["left"] != -1).sum() >= cfg["rounds"], "the trees should really split"
    assert replayed.keys() == direct.keys()
    for k in replayed:
        np.testing.assert_array_equal(replayed[k], direct[k], err_msg=k)
