// text_parse.h -- the byte-level code of the device text parsers (csv.cu): field literals, newline counting and the libsvm
// token walk.  Under nvcc every function is __host__ __device__; under g++ they are plain inline functions, so
// tests/helpers/text_parse_sweep.cc checks exactly the code the kernels run.
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define B200_TEXT_FN __host__ __device__ __forceinline__
#define B200_TEXT_HD __host__ __device__
#else
#define B200_TEXT_FN inline
#define B200_TEXT_HD
#endif

namespace b200 {

B200_TEXT_FN float text_float_from_bits(uint32_t u) { float f; memcpy(&f, &u, sizeof f); return f; }

B200_TEXT_FN int text_popcount(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}

// '\n' bytes in a little-endian word.  The exact zero-byte mask of x = word ^ 0x0a0a0a0a: bit 7 of a byte is set iff the byte
// is zero.  The shorter (x - 0x01010101) & ~x & 0x80808080 only tells whether SOME byte is zero: a borrow out of a '\n' byte
// also sets the bit of a '\v' byte above it ("\n\v" counted twice).
B200_TEXT_FN int newlines_in_word(uint32_t word) {
  const uint32_t x = word ^ 0x0a0a0a0au;
  return text_popcount(~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu));
}

// field whitespace of the fast path; Python's float() strips more ('\v', '\f', Unicode spaces): those take the host route
B200_TEXT_FN bool is_space(char c) { return c == ' ' || c == '\t' || c == '\r'; }

B200_TEXT_FN char lower(char c) { return (c >= 'A' && c <= 'Z') ? (char)(c + 32) : c; }

// Parse [p, e) as a Python-float literal into float32 with the two roundings of the container's route: text -> nearest double
// -> nearest float32.  Clinger's exact fast path: the first 19 significant digits (no non-zero digit after them) form a
// mantissa below 2^53, and with the decimal point moved behind it the exponent is within +-22, so one correctly rounded IEEE
// multiply or divide by an exact power of ten gives the nearest double.  Also taken: the empty field (NaN; a blank one is not), nan / inf /
// infinity in any case with an optional sign, and zero with any exponent.  Returns false when the token is malformed or outside
// the fast path: the host parser decides those.
B200_TEXT_HD inline bool parse_field(const char* p, const char* e, float* out) {
  if (p == e) { *out = text_float_from_bits(0x7fc00000u); return true; }          // empty field -> NaN (encoder.py:31-32)
  while (p < e && is_space(*p)) ++p;
  while (e > p && is_space(e[-1])) --e;
  if (p == e) return false;                                                       // blank but not empty: float(' ') raises
  bool neg = false;
  if (*p == '+' || *p == '-') { neg = *p == '-'; ++p; if (p == e) return false; }
  const int64_t len = e - p;
  if (len == 3 && lower(p[0]) == 'n' && lower(p[1]) == 'a' && lower(p[2]) == 'n') { *out = text_float_from_bits(0x7fc00000u); return true; }
  if ((len == 3 && lower(p[0]) == 'i' && lower(p[1]) == 'n' && lower(p[2]) == 'f') ||
      (len == 8 && lower(p[0]) == 'i' && lower(p[1]) == 'n' && lower(p[2]) == 'f' && lower(p[3]) == 'i' && lower(p[4]) == 'n' && lower(p[5]) == 'i' &&
       lower(p[6]) == 't' && lower(p[7]) == 'y')) { *out = text_float_from_bits(neg ? 0xff800000u : 0x7f800000u); return true; }
  // exp10 is exact for literals shorter than 10^9 bytes: a fraction of many leading zeros and a large written exponent can
  // cancel, so the written exponent saturates only far beyond anything the digits can offset
  unsigned long long mant = 0; int sig = 0; int exp10 = 0; bool any = false, dropped = false;
  while (p < e && *p >= '0' && *p <= '9') {
    any = true;
    if (sig < 19) { mant = mant * 10ull + (unsigned)(*p - '0'); if (mant != 0) ++sig; } else { ++exp10; if (*p != '0') dropped = true; }
    ++p;
  }
  if (p < e && *p == '.') {
    ++p;
    while (p < e && *p >= '0' && *p <= '9') {
      any = true;
      if (sig < 19) { mant = mant * 10ull + (unsigned)(*p - '0'); if (mant != 0) ++sig; --exp10; } else if (*p != '0') dropped = true;
      ++p;
    }
  }
  if (!any) return false;
  if (p < e && (*p == 'e' || *p == 'E')) {
    ++p; bool eneg = false;
    if (p < e && (*p == '+' || *p == '-')) { eneg = *p == '-'; ++p; }
    if (p == e) return false;
    int ev = 0;
    while (p < e && *p >= '0' && *p <= '9') { if (ev < 100000000) ev = ev * 10 + (*p - '0'); ++p; }
    exp10 += eneg ? -ev : ev;
  }
  if (p != e) return false;                                                       // trailing junk (Python's float() would raise)
  if (mant == 0) { *out = neg ? -0.0f : 0.0f; return true; }
  if (dropped || mant >= (1ull << 53) || exp10 > 22 || exp10 < -22) return false;   // outside the exact fast path: host parser decides
  const double p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
  double d = (double)mant;                                                        // exact: mant < 2^53
  d = exp10 >= 0 ? d * p10[exp10] : d / p10[-exp10];                              // one correctly rounded IEEE operation
  *out = (float)(neg ? -d : d);
  return true;
}

// One libsvm line [p, e) ("label idx:val idx:val ..."): emit(idx, val) for every entry in order, where emit returns false when
// the caller's own check fails.  Returns false when the host route must decide the line: an index that is not 1 ... 9 plain
// digits, a value that is empty, outside the fast path or padded with spaces, a second ':' or a '_' in the value.  Tokens are
// separated by ' ' (serve_utils splits on ' ' only) or, with whitespace_mode, also by '\t', '\r', '\f', '\v' (the encoder
// splits on any whitespace).  A token without ':' is the label, or junk both routes ignore.
template <class Emit>
B200_TEXT_HD inline bool libsvm_line(const char* p, const char* e, int whitespace_mode, Emit&& emit) {
  bool good = true;
  const char* q = p;
  while (q < e) {
    while (q < e && (*q == ' ' || (whitespace_mode && (*q == '\t' || *q == '\r' || *q == '\f' || *q == '\v')))) ++q;
    const char* t = q;
    while (q < e && !(*q == ' ' || (whitespace_mode && (*q == '\t' || *q == '\r' || *q == '\f' || *q == '\v')))) ++q;
    if (t == q) break;
    const char* c = t; while (c < q && *c != ':') ++c;
    if (c == q) continue;
    int idx = 0; bool ok = c > t && (c - t) <= 9;
    for (const char* d = t; d < c && ok; ++d) { if (*d < '0' || *d > '9') ok = false; else idx = idx * 10 + (*d - '0'); }
    const char* v = c + 1;
    for (const char* d = v; d < q && ok; ++d) if (*d == ':' || *d == '_') ok = false;
    float val = 0.f;
    if (ok) { if (v == q || !parse_field(v, q, &val)) ok = false; else if (v < q && (is_space(*v) || is_space(q[-1]))) ok = false; }
    if (!ok) { good = false; continue; }
    if (!emit(idx, val)) good = false;
  }
  return good;
}

}  // namespace b200
