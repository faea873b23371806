"""Per-round time of reg:squarederror three ways on the same data (default 10M x 28, depth 6), in one call: the built-in
objective, the same loss as a numpy `obj` (g = m - y, h = 1 in float32), and the same loss computed by torch on the device and
handed to Booster.boost in place.  The numpy round is split into the margin copy to the host, the Python objective, and boost()
(the copy of the pairs to the device, the ingest kernel and growth); the torch round into the objective and boost().  Times
are host clocks around work ending in a device synchronise, medians over the timed rounds after the same warm-up rounds.  The
ingest kernel's own time comes from torch.profiler over a separate run of rounds, with its bandwidth over 16 B per row
(8 read, 8 written).

    python microbench/custom_objective_round.py [--rows 10000000] [--cols 28] [--depth 6] [--warmup 2] [--rounds 5]

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
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--cols", type=int, default=28)
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
    g.manual_seed(71)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    y_dev = x @ beta + 0.1 * torch.randn(a.rows, generator=g, device="cuda")
    y = y_dev.cpu().numpy().astype(np.float32)
    d = xgb.DMatrix(x, label=y)
    del x
    params = dict(tree_method="hist", objective="reg:squarederror", max_depth=a.depth, eta=0.3, max_bin=256, seed=1, base_score=0.5)
    sync = be.synchronize

    def run(step):
        bst = xgb.Booster(params, [d])
        parts = []
        for r in range(a.warmup + a.rounds):
            sync(); t0 = time.perf_counter()
            p = step(bst, r)
            sync(); t1 = time.perf_counter()
            if r >= a.warmup:
                parts.append([(t1 - t0) * 1e3] + p)
        return [float(v) for v in np.median(np.array(parts), axis=0)], bst

    def builtin(bst, r):
        bst.update(d, r)
        return []

    def numpy_obj(bst, r):
        t0 = time.perf_counter()
        m = be.booster_training_margin(bst.handle, d.handle)[:, 0]
        t1 = time.perf_counter()
        gr, he = m - y, np.ones_like(m)
        t2 = time.perf_counter()
        bst.boost(d, r, gr, he)
        sync(); t3 = time.perf_counter()
        return [(t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3]

    def torch_boost(bst, r):
        # the margin stays a device quantity a real objective would hold; here it is the torch copy of the cache's margin
        m = torch.from_numpy(be.booster_training_margin(bst.handle, d.handle)[:, 0]).cuda()
        sync(); t0 = time.perf_counter()
        gr, he = m - y_dev, torch.ones_like(m)
        torch.cuda.synchronize(); t1 = time.perf_counter()
        bst.boost(d, r, gr, he)
        sync(); t2 = time.perf_counter()
        return [(t1 - t0) * 1e3, (t2 - t1) * 1e3]

    out = {"rows": a.rows, "cols": a.cols, "depth": a.depth, "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    (b_ms,), b1 = run(builtin)
    out["builtin_round_ms"] = round(b_ms, 3)
    (n_ms, n_d2h, n_py, n_boost), b2 = run(numpy_obj)
    out.update(numpy_obj_round_ms=round(n_ms, 3), numpy_margin_d2h_ms=round(n_d2h, 3), numpy_python_ms=round(n_py, 3), numpy_boost_ms=round(n_boost, 3))
    (t_ms, t_obj, t_boost), b3 = run(torch_boost)
    out.update(torch_boost_round_ms=round(t_ms, 3), torch_objective_ms=round(t_obj, 3), torch_boost_ms=round(t_boost, 3))
    out["numpy_model_equals_builtin"] = b1.save_raw("ubj") == b2.save_raw("ubj")
    out["torch_model_equals_builtin"] = b1.save_raw("ubj") == b3.save_raw("ubj")
    # the ingest kernel alone, from a profiled run of torch rounds
    from torch.profiler import ProfilerActivity, profile
    bst = xgb.Booster(params, [d])
    m = torch.full((a.rows,), 0.5, device="cuda")
    gr, he = (m - y_dev).contiguous(), torch.ones_like(m)
    for r in range(2):
        bst.boost(d, r, gr, he)
    sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(2, 7):
            bst.boost(d, r, gr, he)
        sync()
    ks = [e for e in prof.events() if e.name.startswith("void b200::custom_gradient_kernel") or "custom_gradient_kernel" in e.name]
    us = [e.device_time for e in ks] if ks and hasattr(ks[0], "device_time") else [e.cuda_time for e in ks]
    if us:
        k_ms = float(np.median(us)) / 1e3
        out["ingest_kernel_ms"] = round(k_ms, 4)
        out["ingest_kernel_GBps"] = round(16.0 * a.rows / (k_ms * 1e-3) / 1e9, 1)
        out["ingest_bytes_per_row"] = 16
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
