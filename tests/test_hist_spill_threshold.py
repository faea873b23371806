"""The spill thresholds of the histogram kernels (hist.cu kSpillThresholdG / kSpillThresholdH): whatever an accumulator keeps
between two overflow checks plus the most one window can add must still fit its 32-bit plane, on both fixed-point grids."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _constants():
    src = open(os.path.join(ROOT, "sagemaker-xgboost-container_b200", "csrc", "hist.cu")).read()
    eng = open(os.path.join(ROOT, "sagemaker-xgboost-container_b200", "csrc", "engine.h")).read()
    g = int(re.search(r"kSpillThresholdG = 1 << (\d+);", src).group(1))
    h = int(re.search(r"kSpillThresholdH = 1u << (\d+);", src).group(1))
    grids = [tuple(map(int, m)) for m in re.findall(r"kGradBits\w* = (\d+), kWindowRows\w* = (\d+);", eng)]
    return 1 << g, 1 << h, grids


def test_spill_thresholds_leave_room_for_one_window():
    spill_g, spill_h, grids = _constants()
    assert sorted(grids) == [(18, 8064), (21, 1008)]
    for bits, window in grids:
        assert (spill_g - 1) + window * (1 << bits) <= 2 ** 31 - 1          # signed G plane, either sign
        assert (spill_h - 1) + window * (1 << (bits + 1)) <= 2 ** 32 - 1    # unsigned H plane (h_q <= 2^(bits+1))


def test_spill_thresholds_are_as_high_as_the_grid_allows():
    """Lower thresholds only cost RED.ADD.64 traffic: a constant hessian quantises to 2^(bits+1) per row, so an H threshold
    of 2^24 spilled most H accumulators every window."""
    spill_g, spill_h, grids = _constants()
    for bits, window in grids:
        assert 2 * spill_g + window * (1 << bits) > 2 ** 31 - 1
        assert 2 * spill_h + window * (1 << (bits + 1)) > 2 ** 32 - 1
