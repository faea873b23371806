"""Time one round's evaluation of the container's own metrics on both routes.

    python microbench/container_metrics.py [--rows 1000000,10000000,50000000] [--out DIR]

For each row count: train a binary:logistic model to 10 and then to 200 rounds; after each, time `Booster.eval_set` on the
training matrix with `configure_feval(names)` (the device route) and with the same closure wrapped in a lambda (the host
route: predict() of the whole model, then scikit-learn).  The engine call alone (the device pass without the finishing) is
timed too.  Prints one JSON line per measurement together with the GPU's name
and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NAMES = ["accuracy", "f1", "rmse", "mae", "r2"]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:     # noqa: BLE001
        return "unknown (%s)" % e


def timed(fn, repeats):
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()                       # eval_set ends with a device-to-host copy and a stream synchronise
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1000000,10000000,50000000")
    ap.add_argument("--features", type=int, default=28)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import sagemaker_xgboost_container_b200 as xgb
    from sagemaker_xgboost_container_b200 import container_metrics as CM
    import container_metrics_reference as R
    mod = sys.modules.setdefault(CM.CONTAINER_MODULE, R)
    fn = mod.configure_feval(NAMES)
    host = lambda p, d: fn(p, d)   # noqa: E731  (not recognised: the host route)
    gpu = gpu_info()
    results = []
    for n in [int(v) for v in args.rows.split(",")]:
        rng = np.random.default_rng(0)
        X = rng.standard_normal((n, args.features), dtype=np.float32)
        y = (X[:, :4].sum(axis=1) + rng.standard_normal(n, dtype=np.float32) > 0).astype(np.float32)
        d = xgb.DMatrix(X, label=y)
        del X
        bst = xgb.Booster(dict(objective="binary:logistic", tree_method="hist", max_depth=6, eta=0.1), [d])
        done = 0
        for rounds in (10, 200):
            for i in range(done, rounds):
                bst.update(d, i)
            done = rounds
            bst.eval_set([(d, "train")], rounds, fn)          # warm-up: scratch and summation plan
            dev = timed(lambda: bst.eval_set([(d, "train")], rounds, fn), 5)
            hst = timed(lambda: bst.eval_set([(d, "train")], rounds, host), 1 if n > 10_000_000 else 2)
            native = timed(lambda: bst.eval_set([(d, "train")], rounds), 5)
            # the engine call alone: the device pass and the copy of its raw results, without the scikit-learn finishing
            engine = timed(lambda: xgb.get_backend().booster_eval_container_metrics(bst.handle, d.handle, NAMES, False), 5)
            # the container metrics' fields only: the engine's own logloss sums in double with atomics
            part = lambda line: [f for f in line.split("\t") if f.split(":")[0][len("train-"):] in NAMES]   # noqa: E731
            same = part(bst.eval_set([(d, "train")], rounds, fn)) == part(bst.eval_set([(d, "train")], rounds, host))
            r = {"rows": n, "rounds": rounds, "metrics": NAMES, "device_route_s": dev[0], "device_route_min_s": dev[1],
                 "host_route_s": hst[0], "native_eval_only_s": native[0], "engine_pass_s": engine[0], "same_log_line": same, "gpu": gpu}
            print(json.dumps(r), flush=True)
            results.append(r)
        del d, bst
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "container_metrics.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
