"""Worker for the 2-GPU ranking test: every rank trains rank:ndcg (weighted, topk) on its share of whole query groups, evaluates
ndcg@5 and map on it, and rank 0 writes the model and the evaluation line; launched with torchrun."""
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
    from test_gpu_ranking import two_rank_data, TWO_RANK_PARAMS
    collective.init_from_env(backend="gloo")
    rank, world = collective.get_rank(), collective.get_world_size()
    X, y, sizes, w = two_rank_data()
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    g0, g1 = rank * len(sizes) // world, (rank + 1) * len(sizes) // world
    a, b = ptr[g0], ptr[g1]
    d = xgb.DMatrix(X[a:b], label=y[a:b], weight=w[g0:g1], group=sizes[g0:g1])
    bst = xgb.train(TWO_RANK_PARAMS, d, num_boost_round=3, verbose_eval=False)
    line = bst.eval_set([(d, "train")], 3)
    if rank == 0:
        bst.save_model(out)
        with open(out + ".eval", "w") as f:
            f.write(line)
    collective.finalize()


if __name__ == "__main__":
    main()
