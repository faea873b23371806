#!/usr/bin/env python
"""Kernel-level timing of the histogram kernels through the C-ABI debug entry point (XGB200BuildHistogramEx):
root pass with the TMA kernel (G+H and G-only) and with the gather kernel, and gathered row subsets (deeper levels).
    python microbench/hist_modes.py --rows 50000000 --cols 100 [--out hist_modes.json]
Algorithmic bytes: rows * (F + 8) for contiguous (g,h) passes, rows * (F + 4) for the G-only root pass (mode 2: it reads the
dense g of constant-hessian training, 4 B per row), rows * (F + 8 + 4) with row ids."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import bench
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    dev = torch.device("cuda", 0)
    ba = argparse.Namespace(rows=a.rows, cols=a.cols, seed=43, objective="reg:squarederror", num_class=0)
    X, y = bench.gen_shard(ba, 0, a.rows, dev)
    d = xgb.DMatrix(X, label=y.cpu().numpy())
    del X
    torch.cuda.empty_cache()
    b = xgb.Booster({"max_bin": 256}, [d])
    rng = np.random.default_rng(1)
    n, F = a.rows, a.cols
    gpair = np.empty((n, 2), np.float32)
    gpair[:, 0] = rng.standard_normal(n, dtype=np.float32)
    gpair[:, 1] = 1.0
    peak = bench.hbm_peak()[0]
    res = []

    def run(label, mode, rows=None):
        m = n if rows is None else len(rows)
        gp = gpair if rows is None else gpair[:m]
        be.build_histogram_ex(b.handle, d.handle, gp, mode=mode, row_ids=rows, repeats=2)          # warm-up
        hist, scales, ms, kernel = be.build_histogram_ex(b.handle, d.handle, gp, mode=mode, row_ids=rows, repeats=a.repeats)
        bytes_ = m * (F + (4 if mode == 2 else 8) + (0 if rows is None else 4))
        r = {"case": label, "kernel": kernel, "rows": m, "ms": ms, "gbs": bytes_ / ms / 1e6, "frac_of_peak": bytes_ / ms / 1e6 / peak,
             "checksum": int(hist[:, :, 0].sum()), "checksum_h": int(hist[:, :, 1].sum())}
        res.append(r)
        print(json.dumps(r), flush=True)

    run("root TMA G+H", 0)
    run("root TMA G-only", 2)
    run("root gather-kernel", 1)
    run("every 2nd row", 0, np.arange(0, n, 2, dtype=np.uint32))
    run("every 4th row", 0, np.arange(0, n, 4, dtype=np.uint32))
    sub = np.sort(rng.choice(n, size=n // 4, replace=False).astype(np.uint32))
    run("random 25% sorted", 0, sub)
    sub = np.sort(rng.choice(n, size=n // 16, replace=False).astype(np.uint32))
    run("random 6% sorted", 0, sub)
    if a.out:
        json.dump({"rows": n, "cols": F, "peak_gbs": peak, "results": res}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
