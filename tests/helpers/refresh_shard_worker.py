"""Worker for the two-GPU refresh test: every rank refreshes the same model on its row shard (int64 node sums all-reduced
inside the engine) and rank 0 writes the refreshed model; launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    model, out, n, F = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from util import synth
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y = synth(n, F, 22, "bin")
    lo, hi = rank * n // world, (rank + 1) * n // world
    d = xgb.DMatrix(X[lo:hi], label=y[lo:hi])
    params = dict(objective="binary:logistic", max_depth=5, eta=0.3, max_bin=256, process_type="update", updater="refresh,prune", gamma=1.0)
    bst = xgb.train(params, d, num_boost_round=4, xgb_model=model, verbose_eval=False)
    if rank == 0:
        bst.save_model(out)
    collective.finalize()


if __name__ == "__main__":
    main()
