"""The device text parsers' byte-level code (csrc/text_parse.h) over a sweep of inputs, without a GPU.

tests/helpers/text_parse_sweep.cc is compiled with g++ (UBSan) against the header csv.cu's kernels execute.  Over about 3M
generated literals (tests/text_parse_reference.py) parse_field must take exactly what the restated fast-path rule takes, give
encoder.py's own float64 -> float32 conversion bit for bit where it does, and never take what Python's float() rejects.
newlines_in_word must count the '\\n' bytes of every one of the 2^32 words; the earlier formula of count_newlines_kernel is
swept beside it and shows its defect (a '\\v' above a '\\n' counted as a second newline).  The libsvm token walk must give,
after the device's assembly, the matrices of both container routes."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import text_parse_reference as R  # noqa: E402


@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    return R.build_helper(tmp_path_factory.mktemp("text_parse"))


@pytest.fixture(scope="module")
def literal_sweep(helper, tmp_path_factory):
    lits = R.generate_literals()
    accepted, values = R.run_literals(helper, tmp_path_factory.mktemp("literals"), lits)
    return lits, accepted, values


def test_the_sweep_is_large_and_reaches_both_outcomes(literal_sweep):
    lits, accepted, _ = literal_sweep
    assert len(lits) > 3_000_000
    assert 1_000_000 < accepted.sum() < len(lits) - 1_000_000


def test_parse_field_takes_exactly_what_the_fast_path_rule_takes(literal_sweep):
    lits, accepted, _ = literal_sweep
    rule = np.array([R.fast_path_accepts(s) for s in lits])
    differ = np.nonzero(rule != accepted)[0]
    assert differ.size == 0, [(lits[i][:40], bool(accepted[i])) for i in differ[:20]]


def test_taken_literals_equal_the_container_conversion_bit_for_bit(literal_sweep):
    lits, accepted, values = literal_sweep
    idx = np.nonzero(accepted)[0]
    want = R.reference_float32([lits[i] for i in idx])
    got = values[idx]
    if not R.same_float32(got, want):
        bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want)))[0]
        pytest.fail("%d literals differ, e.g. %r" % (bad.size, [(lits[idx[i]][:40], float(got[i]), float(want[i])) for i in bad[:10]]))


def test_nothing_float_rejects_is_taken(literal_sweep):
    lits, accepted, _ = literal_sweep
    taken_but_invalid = [s for s, a in zip(lits, accepted) if a and not R.float_accepts(s)]
    assert taken_but_invalid == []


@pytest.mark.parametrize("lit,taken", [
    ("9007199254740991", True), ("9007199254740992", False), ("9007199254740993", False),
    ("1e22", True), ("1e23", False), ("1e-22", True), ("1e-23", False),
    ("0.001e25", True), ("0.001e26", False), ("1234.5e23", True), ("1234.5e24", False), ("1234.5e-21", True), ("1234.5e-22", False),
    ("1234567890123456789", False), ("123456789012345678", False), ("1234567890123456", True), ("1234567890123456789e-10", False),
    ("12345678901234567.00", False), ("1.00000000000000", True), ("1.000000000000000000", False), ("0.12345678901234567890", False),
    pytest.param("0." + "0" * 1000010 + "1e1000005", True, id="1e-6-as-1MB"),   # leading fraction zeros cancel a 7-digit exponent
    ("", True), (" ", False), ("\t\r", False), (" 1.5\r", True), ("\v1.5", False), ("1.5\f", False),
    ("-nan", True), ("+InFiNiTy", True), ("infinit", False), ("0e99999", True), ("-0", True),
    ("1_000", False), ("0x10", False), ("١٢", False), ("1e400", False), ("e5", False), ("1e", False), ("+", False),
    (".", False), ("1.2.3", False), ("--1", False), ("1e5e5", False), (".5", True), ("5.", True), ("1E+05", True),
])
def test_named_literals(helper, tmp_path, lit, taken):
    accepted, values = R.run_literals(helper, tmp_path, [lit])
    assert bool(accepted[0]) == taken == R.fast_path_accepts(lit)
    if taken:
        assert R.same_float32(values, R.reference_float32([lit]))


def test_newline_count_is_exact_on_every_word(helper):
    w = R.run_words(helper)
    assert w["words"] == 2 ** 32
    assert w["new_bad"] == 0, "newlines_in_word miscounts %d words, first %#010x" % (w["new_bad"], w["new_first_bad"])
    # the earlier formula: the sweep reaches its defect; the first word it gets wrong is the bytes "\n\v"
    assert w["old_bad"] == 196_607 and w["old_first_bad"] == 0x00000B0A


# ------------------------------------------------------------------------------------------------------------- libsvm
def _libsvm_bodies():
    import test_gpu_serving as T
    bodies = []
    for seed in range(6):
        rng = np.random.default_rng(100 + seed)
        for one_based in (True, False):
            bodies.append(T._libsvm_body(rng, 300, 40, one_based, fmt=("%.6g", "%.9g", "%.3e")[seed % 3]))
    bodies += [
        T._libsvm_body(np.random.default_rng(99), 300, 40, True, fmt="%.17g"),   # mostly outside the fast path: host route
        "1 1:0.5 1:0.25 2:3",                      # repeated index: the sparse route sums it, the dense route keeps the last
        "1 1:2:3 2:4", "1 1:2 2:3:4",              # ':' inside a value
        "1 1:2\r\n0 2:3\r\n1 3:4",                 # CRLF
        "1 1:2\t3:4 5:6", "0\t1:2\t2:3\n1\t3:4",   # tabs
        "1 1:2\n\v0 2:3", "1 1:2\n\f0 2:3", "1 1:2\n\t0 2:3", "1 1:2\n\r0 2:3", "1 1:2\n 0 2:3",
        "1 0:1 5:2\n0 2:3", "1 1:1 5:2\n0 2:3",    # 0-based and 1-based
        "1 1:1e3 2:-0 3:+.5 4:5. 5:1E-5", "1 1:inf 2:-inf", "1 1:nan 2:3",
        "1 1:1_0 2:3", "1 1: 2:3", "1 :1 2:3", "1 a:1 2:3", "1 +1:0.5 2:3", "1 1:0x10",
        "1 1:0.12345678901234567890123 2:3", "1 1:2\n0\n1 4:1", "1\n0 1:2", "0 3:1e-3\t7:2 \n\n1 1:5",
    ]
    return [b.strip() for b in bodies]


@pytest.mark.parametrize("mode", [0, 1])
def test_libsvm_walk_gives_both_container_routes(helper, tmp_path, mode):
    import test_gpu_serving as T
    bodies = _libsvm_bodies()
    walked = R.run_libsvm(helper, tmp_path, bodies, mode)
    ref = T._ref_sparse_route if mode == 0 else T._ref_dense_route
    statuses = []
    for body, lines in zip(bodies, walked):
        assert len(lines) == body.count("\n") + 1
        st, got = R.device_libsvm_matrix(lines, mode)
        statuses.append(st)
        if st == 0:
            want = ref(body)
            assert R.same_float32(got, want), body[:80]
    assert statuses[:12] == [0] * 12                                  # the random bodies all stay on the device
    named = dict(zip(bodies[12:], statuses[12:]))
    assert named["1 1:2:3 2:4"] == named["1 +1:0.5 2:3"] == named["1 1: 2:3"] == named["1 1:1_0 2:3"] == 2
    # the sparse route sums a repeated index and keeps NaN apart; a '\r' before the newline stays in the sparse route's value
    assert named["1 1:0.5 1:0.25 2:3"] == named["1 1:nan 2:3"] == named["1 1:2\r\n0 2:3\r\n1 3:4"] == (2 if mode == 0 else 0)
    assert named["1 1:2\n\v0 2:3"] == named["1 0:1 5:2\n0 2:3"] == named["1 1:inf 2:-inf"] == 0


def test_libsvm_index_digits(helper, tmp_path):
    """Up to nine index digits stay on the device, ten take the host route (the walk's int would overflow)."""
    bodies = ["1 123456789:1.5 1:2", "1 1234567890:1.5 1:2", "1 000000001:2", "1 0000000001:2"]
    for mode in (0, 1):
        walked = R.run_libsvm(helper, tmp_path, bodies, mode)
        assert walked[0] == [(True, [(123456789, 1.5), (1, 2.0)])]
        assert walked[1][0][0] is False and walked[3][0][0] is False
        assert walked[2] == [(True, [(1, 2.0)])]
        assert not any(math.isnan(v) for _, ent in walked[0] for _, v in ent)
