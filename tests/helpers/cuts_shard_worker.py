"""Worker for the 2-GPU cut test: every rank loads its half of the rows with their weights and derives the cuts through the
multi-GPU recipe (capped summaries, all-gathered and merged); rank 0 writes them.  Launched with torchrun."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out = sys.argv[1]
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from test_gpu_cuts import _rank_data
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, w = _rank_data(60_000, 5, 0, 31)
    n = len(X)
    a, b = rank * n // world, (rank + 1) * n // world
    d = xgb.DMatrix(X[a:b], weight=w[a:b])
    p, v, m, _ = xgb.get_backend().dmatrix_get_cuts(d.handle, 256)
    if rank == 0:
        np.savez(out, p=p, v=v, m=m)
    collective.finalize()


if __name__ == "__main__":
    main()
