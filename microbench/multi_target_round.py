"""Per-round time of a multi-target reg:squarederror model with T = 1, 2, 4 and 8 label columns against T single-target models
trained on the columns one by one (the way to fit T targets before multi-target labels), on the same data (default 1M x 100,
depth 6), in one call.  Time is a host clock around Booster.update ending in a device synchronise, the median over the timed
rounds after the same warm-up rounds.

    python microbench/multi_target_round.py [--rows 1000000] [--cols 100] [--depth 6] [--warmup 2] [--rounds 5] [--targets 1,2,4,8]

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--depth", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--targets", default="1,2,4,8")
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    Ts = [int(t) for t in a.targets.split(",")]
    g = torch.Generator(device="cuda")
    g.manual_seed(61)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, max(Ts), generator=g, device="cuda") / (a.cols ** 0.5)
    Y = (x @ beta + 0.1 * torch.randn(a.rows, max(Ts), generator=g, device="cuda")).cpu().numpy().astype(np.float32)
    d = xgb.DMatrix(x, label=Y[:, 0])
    params = dict(tree_method="hist", objective="reg:squarederror", max_depth=a.depth, eta=0.3, max_bin=256, seed=1)

    def round_ms(label):
        d.set_label(label)
        bst = xgb.Booster(params, [d])
        for r in range(a.warmup):
            bst.update(d, r)
        ms = []
        for r in range(a.warmup, a.warmup + a.rounds):
            be.synchronize(); t0 = time.perf_counter()
            bst.update(d, r)
            be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ms)), ms

    out = {"rows": a.rows, "cols": a.cols, "depth": a.depth, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    single = [round_ms(np.ascontiguousarray(Y[:, j]))[0] for j in range(max(Ts))]
    out["single_target_round_ms"] = [round(v, 3) for v in single]
    for T in Ts:
        med, ms = round_ms(np.ascontiguousarray(Y[:, :T]))
        out["T%d_round_ms" % T] = round(med, 3)
        out["T%d_round_ms_all" % T] = [round(v, 3) for v in ms]
        out["T%d_separate_models_round_ms" % T] = round(sum(single[:T]), 3)
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
