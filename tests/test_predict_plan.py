"""The predictor's host-side plan (csrc/predict_plan.h) over a sweep of shapes, without a GPU.

tests/helpers/predict_plan_sweep.cc is compiled with g++ against the header launch_predict executes.  It plans F = 1 ... 40000
(every F up to 1400) against models of stumps, single splits, the fixed slots of trained trees of depth 1 ... 16 and random
tight node counts, 1 ... 400 trees, iteration ranges, matrices wider and narrower than the model, children adjacent or not.
Every tiled plan must run: 32 ... 1024 rows per tile, <= 220 KB of shared memory, chunks within the node budget that tile the
tree range with no gap.  Where the earlier arithmetic was sound the plan must not have changed; where it was not, the sweep
shows it: a tile of zero rows (a division by zero on the host) for full chunks at F = 980 ... 1247, and the tiled kernel on
matrices narrower than the model (it reads the features the matrix lacks from the pad column or the next row).
"""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sagemaker-xgboost-container_b200", "csrc")


@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path_factory.mktemp("plan") / "sweep")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-fsanitize=undefined", "-I", CSRC,
           os.path.join(ROOT, "tests", "helpers", "predict_plan_sweep.cc"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, UBSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0 and not r.stderr, (r.stdout + r.stderr)[-3000:]
    return json.loads(r.stdout)


def test_every_plan_can_run(sweep):
    assert sweep["violations"] == []
    assert sweep["plans"] > 5_000_000
    # every branch is reached: tiled with one and with several chunks, 32-row tiles, each reason for thread-per-row
    assert sweep["tiled"] > 1_000_000 and sweep["multi_chunk"] > 100_000 and sweep["min_rows_chunks"] > 1000
    assert set(sweep["reasons"]) == {"B200XGB_PREDICT_LEGACY", "children not adjacent", "matrix narrower than the model",
                                     "rows too wide", "tree too large"}


def test_plans_the_earlier_arithmetic_got_right_are_unchanged(sweep):
    assert sweep["compared"] > 1_000_000
    assert sweep["changed_where_sound"] == 0


def test_the_sweep_reaches_both_defects_of_the_earlier_arithmetic(sweep):
    """Zero-row tiles once a chunk is full: F = 988 ... 1247 for depth-6 slots, 992 ... 1247 for depth 8 and 10; 95 depth-6
    trees at F = 1000, 64 at F = 1247.  And the tiled kernel on matrices narrower than the model."""
    z = sweep["parent_zero_row_f"]
    assert z["depth6"] == [988, 1247] and z["depth8"] == [992, 1247] and z["depth10"] == [992, 1247]
    assert sweep["parent_first_zero_depth6"] == {"1000": 95, "1247": 64}
    assert sweep["parent_narrow_tiled"] > 0


def test_config5_plan(sweep):
    """BASELINE config 5 (28 features, 50 trees of depth 6): one chunk of 1024-row tiles, as before."""
    assert sweep["config5"] == {"kernel": "predict_tiled_kernel", "reason": "", "has_nan": False, "tree_begin": 0, "tree_end": 50,
                                "pitch": 29, "chunks": [{"begin": 0, "end": 50, "node_bytes": 51200, "rows": 1024, "threads": 1024,
                                                         "smem": 170192}]}
