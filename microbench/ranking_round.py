"""Rounds of rank:ndcg, rank:pairwise, rank:map and reg:squarederror on one synthetic learning-to-rank shape (10M x 136, query
groups of uniform size in [1, 240], about 83k of them, labels 0-4, depth 6), then rank:ndcg on a second shape with groups of 10k
rows and on a third with no groups (one group of every row), in one call:

  - the wall time (host clock around Booster.update ending in a device synchronise) of one round of each objective after the
    same warm-up rounds; rank:ndcg and rank:map (binary labels) run the topk pairs with K = 32, rank:pairwise the mean pairs with
    K = 1 (lambdarank_pair_method=mean);
  - the gradient stage of one more rank:ndcg round (torch.profiler with CUDA activities): the summed time of the ranking kernels
    (the segmented sort of the margins, rank.cu's kernels) against the summed time of every other kernel of the round (tree
    growth), and the pairs evaluated per second.  A pair (i, j) with i < min(K, n), i < j is evaluated once from each end.

    python microbench/ranking_round.py [--rows 10000000] [--cols 136] [--warmup 2] [--rounds 3] [--large-group 10000]

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
RANK_KERNELS = ("key_kernel", "position_kernel", "rank_mean_kernel", "unfix_kernel", "DeviceSegmentedSort", "DeviceSegmentedRadixSort", "DeviceSegmentedSortKernel", "gather_labels_kernel",
                "map_prefix_kernel", "inv_idcg_kernel", "rank_pairs_kernel", "group_scale_kernel", "rank_write_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def pairs_evaluated(sizes, K):
    import numpy as np
    n = sizes.astype(np.int64)
    kk = np.minimum(n, K)
    return int(2 * np.sum(kk * n - kk * (kk + 1) // 2))        # sum over i < kk of (n - 1 - i), from each end


def time_rounds(xgb, be, d, params, warmup, rounds):
    import numpy as np
    bst = xgb.Booster(params, [d])
    for r in range(warmup):
        bst.update(d, r)
    ms = []
    for r in range(warmup, warmup + rounds):
        be.synchronize(); t0 = time.perf_counter()
        bst.update(d, r)
        be.synchronize(); ms.append((time.perf_counter() - t0) * 1e3)
    return bst, round(float(np.median(ms)), 3)


def profile_round(bst, be, d, it):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bst.update(d, it)
        be.synchronize()
    rank = other = 0.0
    for e in prof.key_averages():
        if e.device_time_total <= 0:
            continue
        if any(k in e.key for k in RANK_KERNELS):
            rank += e.device_time_total
        else:
            other += e.device_time_total
    return rank / 1e3, other / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--cols", type=int, default=136)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--large-group", type=int, default=10_000)
    a = ap.parse_args()
    import numpy as np
    import torch
    import sagemaker_xgboost_container_b200 as xgb
    be = xgb.get_backend()
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(53)
    x = torch.randn(a.rows, a.cols, generator=g, device="cuda", dtype=torch.float32)
    x = torch.round(torch.clamp(x, -4.0, 4.0 - 1.0 / 32) * 32) / 32
    beta = torch.randn(a.cols, generator=g, device="cuda") / (a.cols ** 0.5)
    score = (x @ beta + 0.5 * torch.randn(a.rows, generator=g, device="cuda")).cpu().numpy()
    d = xgb.DMatrix(x, label=np.zeros(a.rows, np.float32))
    del x
    torch.cuda.empty_cache()
    rng = np.random.default_rng(53)
    sizes = rng.integers(1, 241, a.rows // 120 + 1000)
    sizes = sizes[:np.searchsorted(np.cumsum(sizes), a.rows)]
    sizes = np.append(sizes, a.rows - sizes.sum())
    graded = np.clip(np.floor(score * 1.2 + 2.0), 0, 4).astype(np.float32)
    binary = (graded >= 3).astype(np.float32)
    base = dict(tree_method="hist", max_depth=6, eta=0.3, max_bin=256, seed=1)
    out = {"rows": a.rows, "cols": a.cols, "groups": int(len(sizes)), "warmup_rounds": a.warmup, "timed_rounds": a.rounds}
    d.set_group(sizes)
    runs = (("reg:squarederror", graded, {}), ("rank:ndcg", graded, {}), ("rank:pairwise", graded, {"lambdarank_pair_method": "mean"}),
            ("rank:map", binary, {}))
    for name, y, extra in runs:
        d.set_label(y)
        bst, ms = time_rounds(xgb, be, d, dict(base, objective=name, **extra), a.warmup, a.rounds)
        key = name.split(":")[1]
        out[key + "_round_ms"] = ms
        out[key + "_rounds_per_s"] = round(1e3 / ms, 2)
        if name == "rank:ndcg":
            rank_ms, other_ms = profile_round(bst, be, d, a.warmup + a.rounds)
            out["ndcg_gradient_stage_ms"] = round(rank_ms, 4)
            out["ndcg_tree_growth_ms"] = round(other_ms, 4)
            out["ndcg_pairs_evaluated"] = pairs_evaluated(sizes, 32)
            out["ndcg_pairs_per_s"] = pairs_evaluated(sizes, 32) / (rank_ms / 1e3) if rank_ms > 0 else None
        del bst
    big = np.full(a.rows // a.large_group, a.large_group)
    big = np.append(big, a.rows - big.sum()) if big.sum() < a.rows else big
    big = big[big > 0]
    d.set_group(big)
    d.set_label(graded)
    bst, ms = time_rounds(xgb, be, d, dict(base, objective="rank:ndcg"), a.warmup, a.rounds)
    rank_ms, other_ms = profile_round(bst, be, d, a.warmup + a.rounds)
    out["large_group_rows"] = a.large_group
    out["large_ndcg_round_ms"] = ms
    out["large_ndcg_rounds_per_s"] = round(1e3 / ms, 2)
    out["large_ndcg_gradient_stage_ms"] = round(rank_ms, 4)
    out["large_ndcg_tree_growth_ms"] = round(other_ms, 4)
    out["large_ndcg_pairs_per_s"] = pairs_evaluated(big, 32) / (rank_ms / 1e3) if rank_ms > 0 else None
    del bst
    d.set_uint_info("group_ptr", [0, a.rows])
    bst, ms = time_rounds(xgb, be, d, dict(base, objective="rank:ndcg"), a.warmup, a.rounds)
    rank_ms, other_ms = profile_round(bst, be, d, a.warmup + a.rounds)
    out["one_group_ndcg_round_ms"] = ms
    out["one_group_ndcg_gradient_stage_ms"] = round(rank_ms, 4)
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
