"""tree_method=approx against hist for binary:logistic (depth 6, max_bin 256, continuous features: every feature has more
distinct values than bins, so every feature is re-sketched before every tree), per shape, in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of a hist round and of an approx round,
    after the same warm-up rounds, and the first approx round (which also builds the matrix's sorted orders once);
  - one more approx round under torch.profiler with CUDA activities, its kernel time split into the re-sketch (approx_*
    kernels), the re-bin (bin_kernel, pad_rows_kernel, transpose_bins_kernel) and the rest (gradient and tree);
  - the re-sketch's bytes per tree from the sketch's shape (each kept entry: 4 B of order + one 32 B sector of the hessian
    gathered by row; each run: its 4 B start, its 8 B weight written, read and rewritten by the scan) over its kernel time,
    against the 3.35 TB/s of HBM3 on NVIDIA's H100 SXM data sheet, and the sketch's resident bytes from the same shape.

    python microbench/approx_round.py [--shapes 1000000x28,10000000x100] [--warmup 2] [--rounds 3]

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
REBIN = ("bin_kernel", "pad_rows_kernel", "transpose_bins_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def one_shape(xgb, be, torch, rows, cols, warmup, rounds):
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    x = torch.randn(rows, cols, generator=g, device="cuda", dtype=torch.float32)
    beta = torch.randn(cols, generator=g, device="cuda") / (cols ** 0.5)
    z = x @ beta + 0.5 * torch.randn(rows, generator=g, device="cuda")
    y = (torch.sigmoid(z) > torch.rand(rows, generator=g, device="cuda")).float().cpu().numpy()
    d = xgb.DMatrix(x, label=y)
    del x, z
    torch.cuda.empty_cache()
    out = {"rows": rows, "cols": cols, "warmup_rounds": warmup, "timed_rounds": rounds}

    def round_ms(bst, it):
        be.synchronize()
        t = time.perf_counter()
        bst.update(d, it)
        be.synchronize()
        return (time.perf_counter() - t) * 1e3

    for tm in ("hist", "approx"):
        bst = xgb.Booster(dict(objective="binary:logistic", tree_method=tm, max_depth=6, eta=0.3, max_bin=256, seed=1), [d])
        first = round_ms(bst, 0)
        for i in range(1, warmup):
            round_ms(bst, i)
        ms = [round_ms(bst, warmup + i) for i in range(rounds)]
        out[tm + "_round_ms"] = round(sorted(ms)[len(ms) // 2], 3)
        out[tm + "_first_round_ms"] = round(first, 3)
        if tm == "approx":
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                bst.update(d, warmup + rounds)
                be.synchronize()
            sk = rb = rest = 0.0
            for e in prof.key_averages():
                us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                if "approx_" in e.key:
                    sk += us
                elif any(k in e.key for k in REBIN):
                    rb += us
                else:
                    rest += us
            out["approx_resketch_kernel_ms"] = round(sk / 1e3, 3)
            out["approx_rebin_kernel_ms"] = round(rb / 1e3, 3)
            out["approx_other_kernel_ms"] = round(rest / 1e3, 3)
            # every feature is kept and (continuous data) nearly every value is its own run
            entries = rows * cols
            runs = entries
            sketch_bytes = entries * (4 + 32) + runs * (4 + 8 * 3)
            out["resketch_model_bytes"] = sketch_bytes
            out["resketch_share_of_hbm"] = round(sketch_bytes / HBM_BYTES_PER_S / (sk / 1e6), 3) if sk > 0 else None
            out["sketch_resident_bytes"] = entries * 4 + runs * (4 + 8)
        del bst
    del d
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1000000x28,10000000x100")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    for s in a.shapes.split(","):
        rows, cols = (int(v) for v in s.split("x"))
        print(json.dumps(one_shape(xgb, be, torch, rows, cols, a.warmup, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
