"""The cost of one evaluation of the AUC family against a training round on the same matrix, in one call:

  - binary `auc` (auc.cu, allocates its scratch per call) and `aucpr` (curve.cu) on 10M x 28 rows of binary:logistic;
  - multi-class `auc` and `aucpr` on 5M x 50 rows of multi:softprob with num_class=10 (BASELINE config 4's shape);
  - each as the median wall time of Booster.eval_set (a host clock; the call ends in the copy of the value to the host)
    over --evals calls after --warmup, and as a fraction of the median time of a training round (depth 6) on that matrix.

    python microbench/auc_eval.py [--binary-rows 10000000] [--multi-rows 5000000] [--warmup 3] [--evals 10]

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


def _median_ms(fn, warmup, reps, sync):
    import numpy as np
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        sync(); t0 = time.perf_counter()
        fn()
        sync(); ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms)), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--binary-rows", type=int, default=10_000_000)
    ap.add_argument("--multi-rows", type=int, default=5_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--evals", type=int, default=10)
    a = ap.parse_args()
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(71)
    out = {"warmup": a.warmup, "evals": a.evals}
    cases = (("binary", a.binary_rows, 28, dict(objective="binary:logistic"), ("auc", "aucpr")),
             ("multi", a.multi_rows, 50, dict(objective="multi:softprob", num_class=10), ("auc", "aucpr")))
    for key, rows, cols, obj, metrics in cases:
        x = torch.randn(rows, cols, generator=g, device="cuda", dtype=torch.float32)
        beta = torch.randn(cols, obj.get("num_class", 1), generator=g, device="cuda")
        z = x @ beta + torch.randn(rows, obj.get("num_class", 1), generator=g, device="cuda")
        y = (z[:, 0] > 0).float() if key == "binary" else torch.argmax(z, dim=1).float()
        d = xgb.DMatrix(x, label=y.cpu().numpy())
        del x, z
        torch.cuda.empty_cache()
        bst = xgb.Booster(dict(tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1, **obj), [d])
        it = [0]

        def step():
            bst.update(d, it[0]); it[0] += 1
        round_ms, rms = _median_ms(step, 2, 5, be.synchronize)
        out[key + "_rows"], out[key + "_cols"] = rows, cols
        out[key + "_round_ms"] = round(round_ms, 3)
        for m in metrics:
            ev = xgb.Booster({"eval_metric": m}, [d], model_file=bst)         # the trained model with this one metric
            t, ms = _median_ms(lambda: ev.eval_set([(d, "v")], it[0]), a.warmup, a.evals, be.synchronize)
            out["%s_%s_eval_ms" % (key, m)] = round(t, 3)
            out["%s_%s_eval_ms_all" % (key, m)] = [round(v, 3) for v in ms]
            out["%s_%s_share_of_round" % (key, m)] = round(t / round_ms, 4)
            out["%s_%s_value" % (key, m)] = ev.eval_set([(d, "v")], it[0]).split(":")[-1]
            del ev
        del bst, d
        torch.cuda.empty_cache()
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
