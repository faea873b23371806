"""Worker for the two-rank custom-objective test: every rank trains on its row shard with a numpy squared-error objective
(its own shard's gradients) and rank 0 writes the model; launched with torchrun."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out, n, F, rounds = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from util import synth
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y = synth(n, F, 21, "reg")
    lo, hi = rank * n // world, (rank + 1) * n // world
    d = xgb.DMatrix(X[lo:hi], label=y[lo:hi])

    def obj(margin, dm):
        return (margin - dm.get_label()).astype(np.float32), np.ones_like(margin, np.float32)
    bst = xgb.train(dict(objective="reg:squarederror", max_depth=5, base_score=0.5), d, num_boost_round=rounds, obj=obj, verbose_eval=False)
    if rank == 0:
        bst.save_model(out)
    collective.finalize()


if __name__ == "__main__":
    main()
