"""One boosted-random-forest round (num_parallel_tree = P) against P gbtree rounds on the headline shape (50M x 100,
reg:squarederror, depth 6, subsample 0.8, colsample_bynode 0.8), in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of one forest round of P trees and of
    P gbtree rounds, both after the same warm-up rounds;
  - the row-sample kernel alone (sample_gpair_kernel, torch.profiler with CUDA activities) in one more forest round: its time
    per tree and the bytes it moves (8 B read + 8 B written per row and class) over that time, against the 3.35 TB/s of HBM3
    on NVIDIA's H100 SXM data sheet.

    python microbench/forest_round.py [--rows 50000000] [--cols 100] [--trees 8] [--warmup 2] [--rounds 3]

Prints the card name and its power limit, then one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--trees", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(43)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    y = (x @ beta + 0.1 * torch.randn(a.rows, generator=g, device="cuda")).cpu().numpy()
    d = xgb.DMatrix(x, label=y)
    del x
    torch.cuda.empty_cache()
    base = dict(objective="reg:squarederror", tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1, subsample=0.8,
                colsample_bynode=0.8)
    P = a.trees
    out = {"rows": a.rows, "cols": a.cols, "trees_per_round": P, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}

    def timed(bst, start, count, per):
        ms = []
        for i in range(count):
            be.synchronize(); t0 = time.perf_counter()
            for r in range(start + i * per, start + (i + 1) * per):
                bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        return ms

    # gbtree: P rounds (P trees) per timed unit; forest: one round of P trees
    for name, params, per in (("gbtree_x%d" % P, base, P), ("forest_P%d" % P, dict(base, num_parallel_tree=P), 1)):
        bst = xgb.Booster(params, [d])
        for r in range(a.warmup * per):
            bst.update(d, r)
        ms = timed(bst, a.warmup * per, a.rounds, per)
        out[name + "_ms"] = [round(v, 3) for v in ms]
        out[name + "_ms_median"] = round(float(np.median(ms)), 3)
        if per == 1:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bst.update(d, a.warmup + a.rounds)
                be.synchronize()
            kus = [e.device_time_total for e in prof.key_averages() if "sample_gpair_kernel" in e.key]
            calls = sum(e.count for e in prof.key_averages() if "sample_gpair_kernel" in e.key)
            total_us = float(sum(kus))
            out["sample_gpair_kernel_calls"] = int(calls)
            if calls:
                per_tree_s = total_us / 1e6 / calls
                moved = 16.0 * a.rows          # K = 1: one float2 read and one written per row
                out["sample_gpair_kernel_ms_per_tree"] = round(per_tree_s * 1e3, 4)
                out["sample_gpair_kernel_bytes_per_s"] = moved / per_tree_s
                out["sample_gpair_kernel_share_of_hbm_peak"] = round(moved / per_tree_s / HBM_BYTES_PER_S, 3)
        del bst
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
