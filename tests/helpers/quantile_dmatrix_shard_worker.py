"""Worker for the 2-GPU QuantileDMatrix test: every rank builds a QuantileDMatrix under the communicator and rank 0 writes the
error it raised; launched with torchrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    out = sys.argv[1]
    import numpy as np
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import collective
    collective.init_from_env(backend="gloo")
    rank = collective.get_rank()
    try:
        xgb.QuantileDMatrix(np.zeros((10, 3), np.float32))
        msg = "no error"
    except xgb.XGBoostError as e:
        msg = str(e)
    if rank == 0:
        with open(out, "w") as f:
            f.write(msg)
    collective.finalize()


if __name__ == "__main__":
    main()
