#!/usr/bin/env python
"""Where a boosting round's device time goes: root histogram pass, deeper histograms, row partition and prediction-cache
update, timed with CUDA events around each launch group (Booster profile mode) on the bench.py workload.
    python microbench/partition_profile.py --rows 50000000 --cols 100 [--out partition_profile.json]
The round time is taken over graph-replayed rounds (as bench.py times them); the profiled rounds that follow are issued
directly so that every launch group can be bracketed.
Partition byte model, as the library reports it for the profiled trees (profile keys part_*).  Depth-wise trees up to
max_depth 7 are routed (route_kernel + route_scan_kernel + scatter_kernel); part_rows counts the rows routed (every row at
every split level), part_rows_written the built children's rows scattered:
  per row at the root level:    1 [split-feature byte] + 1 [node id written] + 1 [node id read by the scatter]
  per row at deeper levels:     1 [node id read] + 3
  per built row (_out):         payload [the round's gradient by row] + tail [by row] + 4 [row id] + payload + tail  [written]
Lossguide and deeper trees move every row of a split node through part_kernel; then part_rows counts the rows of split
nodes read and part_rows_written the rows written:
  read at the root level:   payload [the round's gradient by row] + tail + 1 [split-feature byte]
  read at deeper levels:    4 [row id] + payload + tail + 1
  written:                  4 + payload + tail
payload = 4 (g alone, constant-hessian objectives, whose round gradients are a dense float g) or 8 ((g,h)); tail = 4 when the rows' 4 tail bin bytes travel with their
ids (a 4-wide tail that the line-aligned row copy does not hold), else 0."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--cols", type=int, default=100)
    ap.add_argument("--max-depth", type=int, default=6)
    ap.add_argument("--objective", default="reg:squarederror")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--timed", type=int, default=10)
    ap.add_argument("--profiled", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import bench
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    dev = torch.device("cuda", 0)
    ba = argparse.Namespace(rows=a.rows, cols=a.cols, seed=43, objective=a.objective, num_class=0)
    X, y = bench.gen_shard(ba, 0, a.rows, dev)
    d = xgb.DMatrix(X, label=y.cpu().numpy())
    del X
    torch.cuda.empty_cache()
    params = bench.params_of(argparse.Namespace(objective=a.objective, max_depth=a.max_depth, max_bin=256, num_class=0))
    b = xgb.Booster(params, [d])
    it = 0
    for _ in range(a.warmup):
        b.update(d, it); it += 1
    be.synchronize()
    be.timer_start()
    for _ in range(a.timed):
        b.update(d, it); it += 1
    round_ms = be.timer_stop() / a.timed
    be.booster_set_profile(b.handle, True)
    for _ in range(a.profiled):
        b.update(d, it); it += 1
    p = be.booster_get_profile(b.handle)
    be.booster_set_profile(b.handle, False)
    R = a.profiled
    root_rows = a.rows * R                        # the root split reads all rows without row ids (every profiled tree splits its root)
    part_bytes = (root_rows * p["part_row_bytes_in_root"] + (p["part_rows"] - root_rows) * p["part_row_bytes_in"] +
                  p["part_rows_written"] * p["part_row_bytes_out"])
    peak = bench.hbm_peak()[0]
    part_gbs = part_bytes / (p["part_ms"] * 1e-3) / 1e9 if p["part_ms"] > 0 else 0.0
    name = torch.cuda.get_device_name(dev)
    try:
        import pynvml
        pynvml.nvmlInit()
        power_w = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        power_w = None
    out = {"gpu": name, "power_limit_w": power_w, "rows": a.rows, "cols": a.cols, "objective": a.objective, "max_depth": a.max_depth, "profiled_rounds": R,
           "round_ms": round_ms,
           "per_round_ms": {"root_hist": p["root_hist_ms"] / R, "deep_hist": p["deep_hist_ms"] / R, "partition": p["part_ms"] / R,
                            "update_margin": p["margin_ms"] / R},
           "per_round_launches": {"root_hist": p["root_hist_launches"] / R, "deep_hist": p["deep_hist_launches"] / R,
                                  "partition": p["part_launches"] / R, "update_margin": p["margin_launches"] / R},
           "partition_share_of_round": p["part_ms"] / R / round_ms,
           "partition_rows_per_round": p["part_rows"] / R, "partition_rows_written_per_round": p["part_rows_written"] / R,
           "partition_row_bytes": {"in_root": p["part_row_bytes_in_root"], "in": p["part_row_bytes_in"], "out": p["part_row_bytes_out"]},
           "partition_bytes_per_round": part_bytes / R, "partition_gbs": part_gbs, "partition_frac_of_peak": part_gbs / peak,
           "peak_gbs": peak, "profile": p}
    print(json.dumps(out), flush=True)
    if a.out:
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
