"""DMatrix against QuantileDMatrix on bench.py's headline regression set (50M x 100, x quantised to 256 levels), in one call:

  - DMatrix from the whole tensor, as bench.py builds it;
  - QuantileDMatrix from a DataIter that generates each 1M-row block (bench.gen_block_torch) when it is asked for.

For each: construction time (host clock around work that ends in a device synchronise), the engine's peak device bytes
(XGB200DeviceMemory: buffers the engine holds, not torch's) during construction and during training, rounds/s over the same
warm-up and timed rounds, the model hash (bench.model_hash), and the predictor kernel's device time over every row (CUDA events,
XGB200BoosterPredictKernelMs): the float predictor on the DMatrix, the bin predictor on the QuantileDMatrix.  Every block has
at most 256 distinct values per feature, under the 2048-point batch summaries, so both constructions have the same cuts and the
two hashes must be equal; the script says so when they are not.

    python microbench/quantile_dmatrix.py [--rows 50000000] [--cols 100] [--warmup 5] [--steps 20]

Prints the card name and its power limit, then one JSON line.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "microbench"))
from absoluteerror_round import card  # noqa: E402
from bench import BLOCK, gen_block_torch, model_hash, params_of  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=43)
    ap.add_argument("--predict-repeats", type=int, default=5)
    a = ap.parse_args()
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    dev = "cuda:0"
    args = argparse.Namespace(objective="reg:squarederror", max_depth=6, max_bin=256, num_class=0)
    params = params_of(args)
    nblocks = (a.rows + BLOCK - 1) // BLOCK

    def block(b):
        return gen_block_torch(b, min(BLOCK, a.rows - b * BLOCK), a.cols, a.seed, "reg:squarederror", 1, dev)

    def run(d):
        torch.cuda.synchronize()
        be.device_memory(reset_peak=True)
        bst = xgb.Booster(params, [d])
        for i in range(a.warmup):
            bst.update(d, i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(a.warmup, a.warmup + a.steps):
            bst.update(d, i)
        torch.cuda.synchronize()
        rps = a.steps / (time.perf_counter() - t0)
        peak = be.device_memory()[1]
        h, ntrees = model_hash(be, bst)
        pred_ms = be.booster_predict_kernel_ms(bst.handle, d.handle, a.predict_repeats)
        return {"rounds_per_sec": rps, "peak_train_bytes": peak, "model_hash": h, "trees": ntrees, "predict_kernel_ms": pred_ms}

    out = {"card": card(), "rows": a.rows, "cols": a.cols, "warmup": a.warmup, "steps": a.steps}

    # DMatrix from the whole tensor (bench.py's construction)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    X = torch.empty((a.rows, a.cols), device=dev, dtype=torch.float32)
    y = torch.empty((a.rows,), device=dev, dtype=torch.float32)
    for b in range(nblocks):
        X[b * BLOCK:(b + 1) * BLOCK], y[b * BLOCK:(b + 1) * BLOCK] = block(b)
    torch.cuda.synchronize()
    be.device_memory(reset_peak=True)
    t1 = time.perf_counter()
    d = xgb.DMatrix(X, label=y.cpu().numpy())
    d_bins = xgb.get_backend().dmatrix_get_cuts(d.handle, 256)      # DMatrix bins lazily: bin here so construction includes it
    torch.cuda.synchronize()
    out["dmatrix"] = {"construct_s": time.perf_counter() - t1, "generate_s": t1 - t0, "peak_construct_bytes": be.device_memory()[1]}
    del X, y, d_bins
    torch.cuda.empty_cache()
    out["dmatrix"].update(run(d))
    del d
    torch.cuda.empty_cache()

    # QuantileDMatrix from a DataIter that generates each block when asked
    class Blocks(xgb.DataIter):
        def __init__(self):
            super().__init__()
            self.b = 0

        def reset(self):
            self.b = 0

        def next(self, input_data):
            if self.b == nblocks:
                return False
            xb, yb = block(self.b)
            input_data(data=xb, label=yb.cpu().numpy())
            self.b += 1
            return True

    torch.cuda.synchronize()
    be.device_memory(reset_peak=True)
    t0 = time.perf_counter()
    q = xgb.QuantileDMatrix(Blocks())
    torch.cuda.synchronize()
    out["quantile_dmatrix"] = {"construct_s": time.perf_counter() - t0, "peak_construct_bytes": be.device_memory()[1],
                               "note": "construct_s includes generating every block twice"}
    torch.cuda.empty_cache()
    out["quantile_dmatrix"].update(run(q))
    same = out["dmatrix"]["model_hash"] == out["quantile_dmatrix"]["model_hash"]
    out["hashes_equal"] = same
    print(out["card"])
    if not same:
        print("MODEL HASHES DIFFER: DMatrix %s, QuantileDMatrix %s" % (out["dmatrix"]["model_hash"], out["quantile_dmatrix"]["model_hash"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
