"""Rounds of survival:aft, survival:cox and reg:squarederror on the headline shape (50M x 100, depth 6), in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of one round of each objective after the
    same warm-up rounds;
  - the Cox gradient stage alone (torch.profiler with CUDA activities, one more Cox round): the summed time of its kernels
    (cox_exp_kernel, the three-phase scans tile_sums / tile_carries / tile_scan, cox_gradient_kernel) and the bytes they move
    over that time, against the 3.35 TB/s of HBM3 on NVIDIA's H100 SXM data sheet.  Bytes per row, counted as the kernels
    request them: exp 16 (order, margin, e), suffix scan 24, (R, S) scan 42 (event, head, D twice, rs written), gradient 37
    (order, e, rs, event, gpair) = 119.

    python microbench/survival_round.py [--rows 50000000] [--cols 100] [--warmup 2] [--rounds 3]

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
COX_BYTES_PER_ROW = 119
COX_KERNELS = ("cox_exp_kernel", "tile_sums_kernel", "tile_carries_kernel", "tile_scan_kernel", "cox_gradient_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(47)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    lin = x @ beta + 0.3 * torch.randn(a.rows, generator=g, device="cuda")
    t = torch.exp(1.0 + 0.5 * lin)
    right = torch.rand(a.rows, generator=g, device="cuda") < 0.3
    lo = t.cpu().numpy()
    hi = torch.where(right, torch.full_like(t, float("inf")), t).cpu().numpy()
    cox_y = torch.where(right, -torch.ceil(t * 50), torch.ceil(t * 50)).cpu().numpy()      # ties and 30 % censored
    y = lin.cpu().numpy()
    d = xgb.DMatrix(x, label=y, label_lower_bound=lo, label_upper_bound=hi)
    del x, lin, t
    torch.cuda.empty_cache()
    base = dict(tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1)
    out = {"rows": a.rows, "cols": a.cols, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    for name in ("reg:squarederror", "survival:aft", "survival:cox"):
        d.set_label(cox_y if name == "survival:cox" else y)
        bst = xgb.Booster(dict(base, objective=name), [d])
        for r in range(a.warmup):
            bst.update(d, r)
        ms = []
        for r in range(a.warmup, a.warmup + a.rounds):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        key = name.split(":")[1]
        out[key + "_round_ms"] = [round(v, 3) for v in ms]
        out[key + "_round_ms_median"] = round(float(np.median(ms)), 3)
        if name == "survival:cox":
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bst.update(d, a.warmup + a.rounds)
                be.synchronize()
            evs = [e for e in prof.key_averages() if any(k in e.key for k in COX_KERNELS)]
            s = float(sum(e.device_time_total for e in evs)) / 1e6
            out["cox_gradient_kernels"] = sorted({e.key.split("(")[0][:60] for e in evs})
            out["cox_gradient_stage_ms"] = round(s * 1e3, 4)
            if s > 0:
                out["cox_gradient_stage_bytes_per_s"] = COX_BYTES_PER_ROW * a.rows / s
                out["cox_gradient_stage_share_of_hbm_peak"] = round(COX_BYTES_PER_ROW * a.rows / s / HBM_BYTES_PER_S, 3)
        del bst
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
