#!/usr/bin/env python
"""Where the time of the device recordio-protobuf path goes: wall time of serving.recordio_protobuf_to_dmatrix on a
1M x 28 dense float32 body and a 1M x 100 sparse body at 10 % density, the stage times of DMatrix::from_recordio (stderr, via
B200XGB_RECORDIO_PROFILE=1: index walk, H2D, passes, scatter), and the package's host route on a slice for comparison.

    python microbench/recordio_stages.py [rows]
"""
import os
import sys
import time

os.environ["B200XGB_RECORDIO_PROFILE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import recordio_reference as R  # noqa: E402
import sagemaker_xgboost_container_b200 as xgb  # noqa: E402,F401
from sagemaker_xgboost_container_b200 import recordio, serving  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
for name, (body, X, y) in (("dense %d x 28 f32" % rows, R.big_dense_body(rows, 28, seed=45)),
                           ("sparse %d x 100 @10%%" % rows, R.big_sparse_body(rows, 100, 10, seed=45))):
    print("== %s: body %.1f MB" % (name, len(body) / 1e6), flush=True)
    best = float("inf")
    for rep in range(4):
        t0 = time.perf_counter()
        d = serving.recordio_protobuf_to_dmatrix(body)
        t1 = time.perf_counter()
        best = min(best, t1 - t0)
        print("recordio_protobuf_to_dmatrix wall %.1f ms (%d x %d)" % ((t1 - t0) * 1e3, d.num_row(), d.num_col()), flush=True)
        del d
    print("best %.1f ms = %.1f M rows/s, %.2f GB/s of body" % (best * 1e3, rows / best / 1e6, len(body) / best / 1e9), flush=True)
    rec_len = len(body) // rows if "dense" in name else None
    n_host = 20_000
    part = body[:n_host * rec_len] if rec_len else R.big_sparse_body(n_host, 100, 10, seed=46)[0]
    t0 = time.perf_counter()
    recordio.read_recordio_protobuf(part)
    t1 = time.perf_counter()
    print("host route on %d rows: %.0f ms = %.0f k rows/s" % (n_host, (t1 - t0) * 1e3, n_host / (t1 - t0) / 1e3), flush=True)
