"""One boosting round at subsample 0.2 under sampling_method=uniform and under sampling_method=gradient_based, in one call, on
50M x 100 reg:squarederror (depth 6, K = 1) and on 5M x 50 multi:softprob (num_class 10):

  - the wall time (host clock around Booster.update ending in a device synchronise) of a round under each method, after the
    same warm-up rounds;
  - in a separate profiled round under gradient_based, the device time of the select kernels (gbs_rag_kernel,
    gbs_hist_kernel, gbs_pick_kernel) and of the sampling kernel (gbs_sample_kernel) from torch.profiler with CUDA activities,
    and their bytes over that time against the 3.35 TB/s of HBM3 on NVIDIA's H100 SXM data sheet.  Bytes per row and class:
    the rag pass reads 8 and writes 4, each of the 4 histogram passes reads 4, the sampling kernel reads 8 and writes 8.

    python microbench/gradient_sampling_round.py [--shape both|reg|softprob] [--warmup 2] [--rounds 3]

Prints the card name and its power limit, then one JSON line per shape.
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
SELECT = ("gbs_rag_kernel", "gbs_hist_kernel", "gbs_pick_kernel")
SHAPES = {"reg": (50_000_000, 100, dict(objective="reg:squarederror")),
          "softprob": (5_000_000, 50, dict(objective="multi:softprob", num_class=10))}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(shape, warmup, rounds):
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    n, F, obj = SHAPES[shape]
    K = obj.get("num_class", 1)
    g = torch.Generator(device="cuda")
    g.manual_seed(44)
    x = torch.randn(n, F, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    if K > 1:
        beta = torch.randn(F, K, generator=g, device="cuda") / (F ** 0.5)
        y = torch.argmax(x @ beta + torch.randn(n, K, generator=g, device="cuda"), dim=1).float().cpu().numpy()
    else:
        beta = torch.randn(F, generator=g, device="cuda") / (F ** 0.5)
        y = (x @ beta + 0.1 * torch.randn(n, generator=g, device="cuda")).cpu().numpy()
    d = xgb.DMatrix(x, label=y)
    del x
    torch.cuda.empty_cache()
    base = dict(obj, tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1, subsample=0.2)
    out = {"shape": shape, "rows": n, "cols": F, "num_class": K, "warmup_rounds": warmup, "timed_rounds": rounds}
    for method in ("uniform", "gradient_based"):
        bst = xgb.Booster(dict(base, sampling_method=method), [d])
        for r in range(warmup):
            bst.update(d, r)
        ms = []
        for r in range(warmup, warmup + rounds):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        out[method + "_round_ms"] = [round(v, 3) for v in ms]
        out[method + "_round_ms_median"] = round(float(np.median(ms)), 3)
        if method == "gradient_based":
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bst.update(d, warmup + rounds)
                be.synchronize()
            ev = prof.key_averages()
            select_us = sum(e.device_time_total for e in ev if any(s in e.key for s in SELECT))
            sample_us = sum(e.device_time_total for e in ev if "gbs_sample_kernel" in e.key)
            select_bytes, sample_bytes = (12.0 + 4 * 4.0) * n * K, 16.0 * n * K
            out["select_ms"] = round(select_us / 1e3, 4)
            out["sample_ms"] = round(sample_us / 1e3, 4)
            if select_us:
                out["select_share_of_hbm_peak"] = round(select_bytes / (select_us / 1e6) / HBM_BYTES_PER_S, 3)
            if sample_us:
                out["sample_share_of_hbm_peak"] = round(sample_bytes / (sample_us / 1e6) / HBM_BYTES_PER_S, 3)
        del bst
    out["card"] = card()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", choices=("both", "reg", "softprob"), default="both")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for shape in (("reg", "softprob") if a.shape == "both" else (a.shape,)):
        run(shape, a.warmup, a.rounds)


if __name__ == "__main__":
    main()
