"""Rounds of reg:absoluteerror against reg:squarederror on the same data (default 10M x 100) at depth 6 (routed levels) and
depth 8, in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of one round of each, after the same
    warm-up rounds, and rounds/s;
  - the leaf refresh's share of an absolute-error round: one more round under torch.profiler with CUDA activities, the summed
    device time of the refresh kernels (leaf numbering, row location, the select passes) over the summed time of all kernels.

    python microbench/absoluteerror_round.py [--rows 10000000] [--cols 100] [--warmup 2] [--rounds 5]

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
REFRESH_KERNELS = ("number_leaves_kernel", "locate_leaves_kernel", "select_hist_kernel", "select_pick_kernel", "select_min_kernel",
                   "select_finish_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(53)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    noise = torch.distributions.Laplace(0.0, 0.5).sample((a.rows,)).to("cuda")
    y = (x @ beta + noise).cpu().numpy()
    d = xgb.DMatrix(x, label=y)
    del x, noise
    torch.cuda.empty_cache()
    out = {"rows": a.rows, "cols": a.cols, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    for depth in (6, 8):
        for name in ("reg:squarederror", "reg:absoluteerror"):
            bst = xgb.Booster(dict(tree_method="hist", max_depth=depth, eta=0.3, max_bin=256, seed=1, objective=name), [d])
            for r in range(a.warmup):
                bst.update(d, r)
            ms = []
            for r in range(a.warmup, a.warmup + a.rounds):
                be.synchronize(); t0 = time.perf_counter()
                bst.update(d, r)
                be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
            key = "%s_depth%d" % (name.split(":")[1], depth)
            med = float(np.median(ms))
            out[key + "_round_ms"] = [round(v, 3) for v in ms]
            out[key + "_rounds_per_s"] = round(1e3 / med, 2)
            if name == "reg:absoluteerror":
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    bst.update(d, a.warmup + a.rounds)
                    be.synchronize()
                evs = prof.key_averages()
                total = float(sum(e.device_time_total for e in evs if e.device_time_total > 0))
                ref = float(sum(e.device_time_total for e in evs if any(k in e.key for k in REFRESH_KERNELS)))
                out[key + "_refresh_ms"] = round(ref / 1e3, 4)
                out[key + "_refresh_share_of_device_time"] = round(ref / total, 4) if total > 0 else None
            del bst
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
