"""Worker for the 2-GPU container-metrics test: every rank trains on its half of the rows with
`custom_metric=configure_feval(names)` and compares, after every round, its device-route values with the container's function
on its own predict(), bit for bit; each rank writes what it saw.  Launched with torchrun."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NAMES = ["accuracy", "f1", "precision_macro", "recall", "rmse", "mae", "r2"]


def main():
    out = sys.argv[1]
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective, container_metrics as CM
    import container_metrics_reference as R
    from util import synth
    mod = sys.modules.setdefault(CM.CONTAINER_MODULE, R)
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y = synth(40000, 8, 21, kind="bin")
    a, b = rank * len(y) // world, (rank + 1) * len(y) // world
    d = xgb.DMatrix(X[a:b], label=y[a:b])
    fn = mod.configure_feval(NAMES)
    seen = {"device": [], "host": []}

    class Compare(xgb.callback.TrainingCallback):
        def after_iteration(self, model, epoch, evals_log):
            seen["device"].append([repr(v) for _, v in CM.evaluate(model, d, NAMES, False)])
            seen["host"].append([repr(v) for _, v in fn(model.predict(d, training=False), d)])
            return False

    xgb.train({"objective": "binary:logistic", "max_depth": 3}, d, num_boost_round=3, evals=[(d, "train")],
              custom_metric=fn, callbacks=[Compare()], verbose_eval=False)
    with open(out + ".%d.json" % rank, "w") as f:
        json.dump(dict(seen, rounds=len(seen["device"])), f)
    collective.finalize()


if __name__ == "__main__":
    main()
