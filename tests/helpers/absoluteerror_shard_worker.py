"""Worker for the 2-GPU reg:absoluteerror test: every rank trains on its row shard (weighted) and rank 0 writes the model;
launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out = sys.argv[1]
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from test_gpu_absoluteerror import TWO_RANK_PARAMS, two_rank_data
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y, w = two_rank_data()
    n = len(y)
    a, b = rank * n // world, (rank + 1) * n // world
    bst = xgb.train(TWO_RANK_PARAMS, xgb.DMatrix(X[a:b], label=y[a:b], weight=w[a:b]), num_boost_round=3, verbose_eval=False)
    if rank == 0:
        bst.save_model(out)
    collective.finalize()


if __name__ == "__main__":
    main()
