"""Update rounds (process_type=update, updater=refresh and refresh,prune) against training rounds on the bench's shape
(default 50M x 100 reg:squarederror) at depth 6, in one call: the wall time (host clock around Booster.update ending in a
device synchronise) of each round, and rounds/s.  The model to update is the one the timed training rounds grew.

    python microbench/refresh_round.py [--rows 50000000] [--cols 100] [--warmup 2] [--rounds 5]

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
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(61)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    y = (x @ beta + 0.1 * torch.randn(a.rows, generator=g, device="cuda")).cpu().numpy()
    d = xgb.DMatrix(x, label=y)
    del x
    torch.cuda.empty_cache()
    params = dict(tree_method="hist", objective="reg:squarederror", max_depth=6, eta=0.3, max_bin=256, seed=1)
    total = a.warmup + a.rounds
    out = {"rows": a.rows, "cols": a.cols, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}

    def timed(bst, label):
        ms = []
        for r in range(total):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize()
            if r >= a.warmup:
                ms.append((time.perf_counter() - t0) * 1e3)
        out[label + "_round_ms"] = [round(v, 3) for v in ms]
        out[label + "_rounds_per_s"] = round(1e3 / float(np.median(ms)), 2)

    bst = xgb.Booster(params, [d])
    timed(bst, "train")
    raw = bst.save_raw("ubj")
    for label, updater in (("refresh", "refresh"), ("refresh_prune", "refresh,prune")):
        up = xgb.Booster(dict(params, process_type="update", updater=updater, gamma=1.0), [d], model_file=bytearray(raw))
        timed(up, label)
        del up
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
