"""booster=dart against gbtree on the headline shape (50M x 100, reg:squarederror, depth 6), in one call:

  - the wall time of a boosting round (host clock around Booster.update ending in a device synchronise) for gbtree and for
    dart (rate_drop 0.1), both after the same warm-up rounds, so that the dart rounds drop a non-trivial set of trees;
  - the dropped-tree margin kernel alone (dart_margin_kernel, torch.profiler with CUDA activities) in one more dart round:
    rows x dropped trees per second, and the bytes of X (rows x F x 4) over the kernel time.

    python microbench/dart_round.py [--rows 50000000] [--cols 100] [--warmup 20] [--rounds 5]

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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rate-drop", type=float, default=0.1)
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
    base = dict(objective="reg:squarederror", tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1)
    out = {"rows": a.rows, "cols": a.cols, "warmup_rounds": a.warmup, "timed_rounds": a.rounds, "rate_drop": a.rate_drop}

    def timed_rounds(bst, start):
        ms = []
        for r in range(start, start + a.rounds):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        return ms

    for name, params in (("gbtree", base), ("dart", dict(base, booster="dart", rate_drop=a.rate_drop))):
        bst = xgb.Booster(params, [d])
        for r in range(a.warmup):
            bst.update(d, r)
        ms = timed_rounds(bst, a.warmup)
        out[name + "_round_ms"] = [round(v, 3) for v in ms]
        out[name + "_round_ms_median"] = round(float(np.median(ms)), 3)
        if name == "dart":
            w_before = be.booster_tree_weights(bst.handle)
            r = a.warmup + a.rounds
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bst.update(d, r)
                be.synchronize()
            w_after = be.booster_tree_weights(bst.handle)[:len(w_before)]
            dropped = int((w_after != w_before).sum())
            kus = sum(e.device_time_total for e in prof.key_averages() if "dart_margin_kernel" in e.key)
            out["dart_dropped_trees_in_profiled_round"] = dropped
            out["dart_trees_with_weight_below_1"] = int((w_after != 1).sum())
            out["dart_margin_kernel_ms"] = round(kus / 1e3, 3)
            if kus > 0:
                s = kus / 1e6
                out["dart_margin_rows_trees_per_s"] = a.rows * dropped / s
                out["dart_margin_x_bytes_per_s"] = a.rows * a.cols * 4 / s
        del bst
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
