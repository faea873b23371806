"""Worker for the 2-GPU survival test: every rank trains survival:aft on its row shard and rank 0 writes the model, then every
rank tries survival:cox and rank 0 records the error; launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out = sys.argv[1]
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from test_gpu_survival import _aft_data
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    n = 40000
    X, lo, hi = _aft_data(n, 10, 29)
    a, b = rank * n // world, (rank + 1) * n // world
    d = xgb.DMatrix(X[a:b], label_lower_bound=lo[a:b], label_upper_bound=hi[a:b])
    bst = xgb.train(dict(objective="survival:aft", max_depth=5, eta=0.3), d, num_boost_round=3, verbose_eval=False)
    if rank == 0:
        bst.save_model(out)
    d.set_label(lo[a:b])
    try:
        xgb.train(dict(objective="survival:cox"), d, num_boost_round=1, verbose_eval=False)
        msg = "trained"
    except xgb.core.XGBoostError as e:
        msg = str(e)
    if rank == 0:
        with open(out + ".cox", "w") as f:
            f.write(msg)
    collective.finalize()


if __name__ == "__main__":
    main()
