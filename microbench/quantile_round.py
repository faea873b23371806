"""Rounds of reg:quantileerror with one and three quantiles against reg:absoluteerror and reg:squarederror on the same data
(default 10M x 100, depth 6), in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of one round of each, after the same
    warm-up rounds, and rounds/s;
  - for the adaptive objectives, the leaf refresh's share of a round: one more round under torch.profiler with CUDA activities,
    the summed device time of the refresh kernels (leaf numbering, row location, the select passes) over that of all kernels.

    python microbench/quantile_round.py [--rows 10000000] [--cols 100] [--depth 6] [--warmup 2] [--rounds 5]

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
from absoluteerror_round import REFRESH_KERNELS, card  # noqa: E402

CASES = (("squarederror", dict(objective="reg:squarederror")), ("absoluteerror", dict(objective="reg:absoluteerror")),
         ("quantile_q1", dict(objective="reg:quantileerror", quantile_alpha="0.5")),
         ("quantile_q3", dict(objective="reg:quantileerror", quantile_alpha="(0.1,0.5,0.9)")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--depth", type=int, default=6)
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
    out = {"rows": a.rows, "cols": a.cols, "depth": a.depth, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    for key, obj in CASES:
        bst = xgb.Booster(dict(tree_method="hist", max_depth=a.depth, eta=0.3, max_bin=256, seed=1, **obj), [d])
        for r in range(a.warmup):
            bst.update(d, r)
        ms = []
        for r in range(a.warmup, a.warmup + a.rounds):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        med = float(np.median(ms))
        out[key + "_round_ms"] = [round(v, 3) for v in ms]
        out[key + "_rounds_per_s"] = round(1e3 / med, 2)
        if key != "squarederror":
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
