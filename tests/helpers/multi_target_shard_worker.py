"""Worker for the two-rank multi-target test: every rank trains on its row shard of a 3-column label (the engine all-reduces
the histograms and the intercept's sums) and rank 0 writes the model; launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out, n, F, rounds, objective = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from test_gpu_multi_target import labels3
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, Y = labels3(n, F, 7, objective)
    lo, hi = rank * n // world, (rank + 1) * n // world
    d = xgb.DMatrix(X[lo:hi], label=Y[lo:hi])
    bst = xgb.train(dict(objective=objective, max_depth=5, eta=0.3, max_bin=256), d, num_boost_round=rounds, verbose_eval=False)
    if rank == 0:
        bst.save_model(out)
    collective.finalize()


if __name__ == "__main__":
    main()
