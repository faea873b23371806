"""In-place prediction against DMatrix + predict, in one call (DESIGN.md "In-place prediction"):

- request-sized host batches: per-call latency of inplace_predict and of DMatrix(X) + predict at 1, 64, 1024 and 65536 rows
  x 28, float32 and float64 numpy (host clock around calls that end in a synchronise, median over the timed calls);
- device inputs: 1M x 28 and 10M x 100 torch CUDA float32 and float64, inplace_predict against DMatrix(t.float().contiguous())
  + predict, and the predictor kernel's achieved bytes per second (the input's bytes over the kernel time torch.profiler
  records for predict_tiled_kernel) against the HBM3 data sheet's 3.35 TB/s;
- a large host batch: 10M x 28 float64 numpy through the chunked staging, against a plain pinned H2D copy of the same bytes.

Every timed inplace result is first checked bit for bit against the DMatrix path.  The models are 50 rounds of depth 6.

    python microbench/inplace_predict.py [--reps 50]

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
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    rng = np.random.default_rng(5)

    def model(F):
        X = rng.standard_normal((200_000, F), dtype=np.float32)
        y = X @ (rng.standard_normal(F).astype(np.float32) / np.sqrt(F))
        return xgb.train(dict(tree_method="hist", max_depth=6, eta=0.3), xgb.DMatrix(X, label=y), 50)

    def same(a_, b_):
        a_ = a_.detach().cpu().numpy() if hasattr(a_, "detach") else a_
        assert np.array_equal(np.asarray(a_, np.float32).view(np.uint32), np.asarray(b_, np.float32).view(np.uint32))

    def median_ms(fn, reps):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
        ts.sort()
        return {"median": ts[len(ts) // 2], "p10": ts[len(ts) // 10], "p90": ts[(9 * len(ts)) // 10]}

    out = {"card": card()}
    b28 = model(28)
    host = {}
    for n in (1, 64, 1024, 65536):
        for dt in ("float32", "float64"):
            X = rng.standard_normal((n, 28)).astype(dt)
            same(b28.inplace_predict(X), b28.predict(xgb.DMatrix(X.astype(np.float32))))
            reps = a.reps if n < 65536 else max(10, a.reps // 5)
            host["%dx28_%s" % (n, dt)] = {"inplace_ms": median_ms(lambda: b28.inplace_predict(X), reps),
                                          "dmatrix_predict_ms": median_ms(lambda: b28.predict(xgb.DMatrix(X)), reps)}
    out["host_batches"] = host

    def kernel_ms(fn):
        from torch.profiler import ProfilerActivity, profile
        fn(); torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        tot = sum(e.device_time_total for e in prof.key_averages() if "predict_tiled_kernel" in e.key)
        return tot / 5 / 1e3

    dev = {}
    b100 = model(100)
    for n, F, b in ((1_000_000, 28, b28), (10_000_000, 100, b100)):
        for dt in (torch.float32, torch.float64):
            t = torch.randn(n, F, device="cuda", dtype=dt)
            ref = b.predict(xgb.DMatrix(t.float().contiguous()))
            same(b.inplace_predict(t), ref)
            reps = 10
            ims = median_ms(lambda: b.inplace_predict(t), reps)
            dms = median_ms(lambda: b.predict(xgb.DMatrix(t.float().contiguous())), reps)
            kms = kernel_ms(lambda: b.inplace_predict(t))
            nbytes = n * F * t.element_size()
            dev["%dx%d_%s" % (n, F, str(dt).split(".")[-1])] = {
                "inplace_ms": ims, "dmatrix_predict_ms": dms, "kernel_ms": kms, "input_bytes": nbytes,
                "kernel_gbs": nbytes / (kms * 1e-3) / 1e9 if kms else None,
                "share_of_3350_gbs": nbytes / (kms * 1e-3) / 3.35e12 if kms else None}
            del t
    out["device_inputs"] = dev

    X = rng.standard_normal((10_000_000, 28))                      # float64 on the host: 2.24 GB
    same(b28.inplace_predict(X[:100000]), b28.predict(xgb.DMatrix(X[:100000].astype(np.float32))))
    ims = median_ms(lambda: b28.inplace_predict(X), 5)
    pinned = torch.from_numpy(X).pin_memory()
    h2d = median_ms(lambda: pinned.to("cuda", non_blocking=True), 5)
    out["large_host_batch"] = {"rows": 10_000_000, "cols": 28, "dtype": "float64", "bytes": X.nbytes, "inplace_ms": ims,
                               "inplace_gbs": X.nbytes / (ims["median"] * 1e-3) / 1e9, "pinned_h2d_ms": h2d,
                               "pinned_h2d_gbs": X.nbytes / (h2d["median"] * 1e-3) / 1e9}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
