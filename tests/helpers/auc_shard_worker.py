"""Worker for the 2-GPU AUC-family test: every rank trains on its half of the rows, evaluates multi-class auc / aucpr and
binary aucpr on it, and writes its predictions; rank 0 writes the evaluation line.  Launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    out = sys.argv[1]
    import numpy as np
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    from test_gpu_auc_family import two_rank_data, TWO_RANK_MULTI, TWO_RANK_BINARY
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y, w, Xb, yb, wb = two_rank_data()
    a, b = rank * len(y) // world, (rank + 1) * len(y) // world
    dm = xgb.DMatrix(X[a:b], label=y[a:b], weight=w[a:b])
    db = xgb.DMatrix(Xb[a:b], label=yb[a:b], weight=wb[a:b])
    bm = xgb.train(TWO_RANK_MULTI, dm, num_boost_round=3, verbose_eval=False)
    bb = xgb.train(TWO_RANK_BINARY, db, num_boost_round=3, verbose_eval=False)
    line = bm.eval_set([(dm, "m")], 3) + "\t" + bb.eval_set([(db, "b")], 3).split("\t", 1)[1]
    np.savez(out + ".%d.npz" % rank, multi=bm.predict(dm).reshape(b - a, -1), binary=bb.predict(db))
    if rank == 0:
        with open(out + ".eval", "w") as f:
            f.write(line)
    collective.finalize()


if __name__ == "__main__":
    main()
