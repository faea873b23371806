"""Reference side of the text-parser tests (csrc/text_parse.h, csrc/csv.cu): the literal generator, a Python restatement of the
device fast path's acceptance rule, the container's own float conversion, and the g++ build of tests/helpers/text_parse_sweep.cc.

The device takes a field when its rule below accepts it and hands the body back to the host route otherwise.  What it takes
must equal encoder.py's `np.array(fields).astype(float)` followed by float32 (xgb.DMatrix of a float64 array), bit for bit."""
import math
import os
import re
import shutil
import struct
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sagemaker-xgboost-container_b200", "csrc")
HELPER = os.path.join(ROOT, "tests", "helpers", "text_parse_sweep.cc")

_NUMBER = re.compile(r"[+-]?([0-9]*)(?:\.([0-9]*))?(?:[eE]([+-]?[0-9]+))?\Z")


def fast_path_accepts(lit):
    """The fast path's rule: the empty field is taken (NaN); otherwise surrounding ' ', '\\t', '\\r' are stripped, and a blank
    field is not taken.  nan / inf / infinity in any ASCII case with an optional sign, and zero with any exponent, are taken;
    otherwise the first 19 significant digits (no non-zero digit after them) form a mantissa < 2^53, and with the decimal
    point moved behind that mantissa the exponent is within +-22."""
    if lit == "":
        return True                                                    # encoder.py maps the empty field to "nan"
    s = lit.strip(" \t\r")
    if s == "" or not s.isascii():
        return False
    word = s[1:] if s[0] in "+-" else s
    if word.lower() in ("nan", "inf", "infinity"):
        return True
    m = _NUMBER.match(s)
    if m is None:
        return False
    whole, frac, exp = m.group(1), m.group(2) or "", m.group(3)
    if whole == "" and frac == "":
        return False
    digits = (whole + frac).lstrip("0")
    if digits == "":
        return True                                                    # zero, whatever the exponent
    mant, dropped = digits[:19], digits[19:]
    if dropped.strip("0"):
        return False
    exp10 = (int(exp) if exp else 0) - len(frac) + len(dropped)
    return int(mant) < 2 ** 53 and -22 <= exp10 <= 22


def float_accepts(lit):
    """What the container's route converts without raising (encoder.py maps the empty field to "nan")."""
    try:
        float(lit or "nan")
        return True
    except ValueError:
        return False


def reference_float32(literals):
    """encoder.py's conversion, np.array(fields).astype(float) with the empty field as "nan", then float32; long literals one
    at a time so the fixed-width string array stays small."""
    literals = [s or "nan" for s in literals]
    short = [i for i, s in enumerate(literals) if len(s) <= 64]
    out = np.empty(len(literals), np.float32)
    with np.errstate(over="ignore"):
        if short:
            out[short] = np.array([literals[i] for i in short]).astype(float).astype(np.float32)
        for i, s in enumerate(literals):
            if len(s) > 64:
                out[i] = np.array([s]).astype(float).astype(np.float32)[0]
    return out


def same_float32(got, want):
    """Bit equality, with NaN compared as NaN only (the device's NaN carries no sign, '-nan' included)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    gn, wn = np.isnan(got), np.isnan(want)
    return got.shape == want.shape and np.array_equal(gn, wn) and np.array_equal(got.view(np.uint32)[~wn], want.view(np.uint32)[~wn])


# ------------------------------------------------------------------------------------------------------------ generator
def _casings(word):
    out = [""]
    for ch in word:
        out = [p + c for p in out for c in (ch.lower(), ch.upper())]
    return out


def _shifted(digits, exp10):
    """`digits` x 10^exp10 written with the decimal point at every position of the digits, and behind leading zeros."""
    out = []
    n = len(digits)
    for i in range(n + 1):
        written = exp10 + (n - i)                                      # point after i digits: (n - i) fraction digits
        text = digits[:i] + "." + digits[i:] if 0 < i < n else (digits if i == n else "0." + digits)
        out.append("%se%d" % (text, written))
    for z in (1, 2, 3):
        out.append("0.%s%se%d" % ("0" * z, digits, exp10 + n + z))
    return out


def generate_literals(seed=2024, n_random=150_000):
    """About 3M literals over every form the fast path has to decide; none contains '\\n'."""
    rng = np.random.default_rng(seed)
    lits = []
    # printf and repr forms of random float32 / float64 values over the whole exponent range (random bit patterns: every
    # exponent, denormals included)
    f32 = rng.integers(0, 2 ** 32, size=n_random, dtype=np.uint64).astype(np.uint32).view(np.float32)
    f64 = rng.integers(0, 2 ** 64 - 1, size=n_random, dtype=np.uint64, endpoint=True).view(np.float64)
    for arr in (f32[np.isfinite(f32)].astype(np.float64), f64[np.isfinite(f64)]):
        for fmt in ("%.6g", "%.9g", "%.17g"):
            lits += [fmt % v for v in arr]
        lits += [repr(float(v)) for v in arr]
    lits += [str(v) for v in f32[np.isfinite(f32)]]                  # float32's own shortest form
    # values of ordinary magnitude: these are mostly inside the fast path
    g = rng.standard_normal(n_random) * np.exp(rng.uniform(-25, 25, n_random))
    for fmt in ("%.6g", "%.9g", "%.17g", "%.3e", "%.9f", "%d"):
        lits += [fmt % (int(v) if fmt == "%d" else v) for v in g]
    lits += [repr(float(v)) for v in g.astype(np.float32)]
    # random digit strings of 1 ... 25 digits, the point anywhere, exponents -30 ... 30
    for _ in range(n_random * 3):
        nd = int(rng.integers(1, 26))
        d = "".join(rng.choice(list("0123456789"), nd))
        cut = int(rng.integers(0, nd + 1))
        body = d[:cut] + ("." + d[cut:] if cut < nd or rng.random() < 0.3 else "")
        if body.startswith(".") and rng.random() < 0.5:
            body = "0" + body
        e = "" if rng.random() < 0.3 else "%s%s%d" % ("eE"[int(rng.integers(0, 2))], ["", "+", "-"][int(rng.integers(0, 3))], int(rng.integers(0, 31)))
        lits.append(["", "+", "-"][int(rng.integers(0, 3))] + body + e)
    # mantissas around 2^53 and 19 / 20 digits, exponents around +-22: through e+-k and through the decimal point
    mants = [2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 1, 5, 12345, 999999999999999, 10 ** 15, 10 ** 16, 4503599627370497,
             1234567890123456789, 9999999999999999999, 10 ** 18, 12345678901234567890, 10 ** 19]
    for m in mants:
        for k in range(-25, 26):
            lits.append("%de%d" % (m, k))
            lits.append("%dE%+d" % (m, k))
            lits.append("-%de%d" % (m, k))
            if len(str(m)) <= 19:
                lits += _shifted(str(m), k)
    lits += ["0.001e25", "0.001e26", "1234.5e19", "1234.5e20", "1234.5e-18", "1234.5e-17", "12345e-23", "1e-22", "1e-23", "1e22", "1e23",
             "10e21", "10e22", "0.1e23", "0.1e24", "100e-24", "100e-25"]
    # float32 midpoints: integers in (2^24, 2^53) halfway between neighbouring float32 values (double rounding cases)
    lo = rng.integers(2 ** 24 + 1, 2 ** 53, size=20_000, dtype=np.uint64).astype(np.float32).astype(np.float64)
    lo = lo[(lo > 2 ** 24) & (lo < 2 ** 53)]
    hi = np.nextafter(lo.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    for a, b in zip(lo, hi):
        mid = (int(a) + int(b)) // 2
        lits += ["%d" % mid, "%d" % (mid + 1), "%d" % (mid - 1)]
        k = int(rng.integers(1, 23))
        lits += ["%de-%d" % (mid, k), "%de+%d" % (mid, k), "%d%se-%d" % (mid, "0" * min(k, 3), min(k, 3))]
        lits.append("%s.%se%d" % (str(mid)[:-3], str(mid)[-3:], 3))
    # float32 midpoints below 2^24 (non-integers), as the nearest double's digits
    f = rng.standard_normal(20_000).astype(np.float32)
    nxt = np.nextafter(f, np.float32(np.inf))
    mids = (f.astype(np.float64) + nxt.astype(np.float64)) / 2
    for v in mids:
        lits += [repr(float(v)), "%.17g" % v, "%.20g" % v, "%.16e" % v]
    # zeros, signs, points, exponent markers
    lits += ["0", "-0", "+0", "00", "000123", "123.000", "0.000123", ".5", "5.", "-.5", "+.5", "-5.", "0.", ".0", "-0.0", "+0.0",
             "0e0", "0e99999", "-0e99999", "0.0e-99999", "0e400", "0e-400", "00000000000000000000000000001", "1E5", "1e+05", "1E-05",
             "1.5E+3", "1e05", "1e0005", "1234567890123456789", "12345678901234567890", "1234567890123456789.0",
             "12345678901234567890e-5", "0.1234567890123456789", "0.12345678901234567890", "0.12345678901234567891",
             "1" + "0" * 25 + "e-20", "1" + "0" * 18, "1" + "0" * 19, "9007199254740992", "9007199254740993", "4.9e-324",
             "2.2250738585072014e-308", "1.7976931348623157e308", "3.4028235e38", "3.4028236e38", "1e39", "1e-45", "1.4e-45",
             "7e-46", "1.17549435e-38", "0." + "0" * 40 + "1e40", "0." + "0" * 30 + "123e30", "0." + "0" * 1000010 + "1e1000005",
             "1" + "0" * 40 + "e-40", "1e-0", "1e+0", "-1e-0"]
    # nan / inf / infinity in every casing, with and without a sign
    for w in ("nan", "inf", "infinity"):
        for c in _casings(w):
            lits += [c, "+" + c, "-" + c]
    # whitespace around literals: the fast path strips ' ', '\t', '\r'; '\v' and '\f' take the host route
    base = ["1.5", "-2e3", "nan", "inf", "0", "", "12345678", ".5", "7."]
    for b in base:
        for left in ("", " ", "\t", "\r", "\v", "\f", " \t", "\r\r"):
            for right in ("", " ", "\t", "\r", "\v", "\f", "\t "):
                lits.append(left + b + right)
    # the host route decides these: digit separators, hex, non-ASCII digits, > 19 significant digits, exponents out of range
    lits += ["1_000", "1_0.5", "1e1_0", "0x10", "0X1p3", "١٢٣", "１２", "1٢", " 1", "1 ",
             "123456789012345678901234567890", "0.123456789012345678901234567890", "1e400", "-1e400", "1e-400", "1e23", "1e-23",
             "1 2", "nan1", "infinit", "infinityy", "in", "na", "abc", "1d5"]
    # malformed
    lits += ["e5", "1e", "+", "-", ".", "1.2.3", "--1", "+-1", "1e5e5", "1e+", "1e-", ".e1", "e", "1.e", "-e5", "0x", "1e5.0",
             "1;5", "+.", "-.", "..5", "5..", "1ee5", "1e++5"]
    for s in lits:
        assert "\n" not in s
    return lits


# ------------------------------------------------------------------------------------------------------------- helper
def build_helper(workdir):
    """tests/helpers/text_parse_sweep.cc against csrc/text_parse.h: g++ -O2 with UBSan, halting on any report."""
    if shutil.which("g++") is None:
        import pytest
        pytest.skip("needs g++")
    exe = os.path.join(str(workdir), "text_parse_sweep")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-fsanitize=undefined", "-pthread", "-I", CSRC, HELPER, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _run(exe, *args, timeout=900):
    r = subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout, env=dict(os.environ, UBSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0 and not r.stderr, (r.stdout + r.stderr)[-3000:]
    return r.stdout


def run_literals(exe, workdir, literals):
    """parse_field on the host over `literals`: (accepted bool array, float32 array)."""
    src, dst = os.path.join(str(workdir), "literals.txt"), os.path.join(str(workdir), "literals.out")
    with open(src, "wb") as f:
        f.write("\n".join(literals).encode("utf-8"))
    _run(exe, "literals", src, dst)
    raw = np.fromfile(dst, np.uint8)
    n = len(literals)
    assert raw.size == 5 * n
    return raw[:n].astype(bool), raw[n:].view(np.uint32).view(np.float32).copy()


def run_words(exe):
    import json
    return json.loads(_run(exe, "words"))


def run_libsvm(exe, workdir, bodies, mode):
    """libsvm_line over every line of every body: per body a list of (good, [(idx, float32), ...]) per line."""
    src, dst = os.path.join(str(workdir), "libsvm%d.txt" % mode), os.path.join(str(workdir), "libsvm%d.out" % mode)
    with open(src, "wb") as f:
        f.write("\0".join(bodies).encode("utf-8"))
    _run(exe, "libsvm", str(mode), src, dst)
    out, cur = [], None
    for line in open(dst):
        tok = line.split()
        if tok[0] == "body":
            cur = []
            out.append(cur)
            continue
        k = int(tok[1])
        ent = [(int(tok[2 + 2 * j]), struct.unpack("<f", struct.pack("<I", int(tok[3 + 2 * j])))[0]) for j in range(k)]
        cur.append((tok[0] == "1", ent))
    assert len(out) == len(bodies)
    return out


def device_libsvm_matrix(lines, mode):
    """What parse_libsvm_device assembles from libsvm_line's per-line results: (status, float32 matrix or None).  Status 0 ok,
    2 host route, 3 no entries; mode 0 fills absent entries with NaN, mode 1 with 0."""
    if not all(good for good, _ in lines):
        return 2, None
    idx = [i for _, ent in lines for i, _ in ent]
    if not idx:
        return 3, None
    if mode == 0 and not lines[-1][1]:
        return 2, None
    shift = 1 if min(idx) >= 1 else 0
    F = max(idx) - shift + 1
    X = np.full((len(lines), F), np.nan if mode == 0 else 0.0, np.float32)
    for r, (_, ent) in enumerate(lines):
        for i, v in ent:
            if mode == 0 and (math.isnan(v) or not math.isnan(X[r, i - shift])):
                return 2, None                                          # NaN value, or an index repeated inside a line
            X[r, i - shift] = v
    return 0, X
