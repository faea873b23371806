// CPU sweep of the text parsers' byte-level code (csrc/text_parse.h), compiled with g++ by tests/test_text_parse_sweep.py.
//
//   text_parse_sweep literals IN OUT       IN: literals separated by '\n'.  OUT: one byte per literal (1 = parse_field took it),
//                                          then the float32 bits of each literal (0 where it was not taken), little-endian.
//   text_parse_sweep words                 newlines_in_word against a byte count over all 2^32 words, and the earlier
//                                          formula of count_newlines_kernel (old_newlines below) against the same count.
//   text_parse_sweep libsvm MODE IN OUT    IN: libsvm bodies separated by '\0'.  OUT: per body a line "body LINES", then per
//                                          line "GOOD K idx bits ..." -- libsvm_line's verdict and entries in whitespace MODE.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <thread>
#include <vector>

#include "text_parse.h"

using namespace b200;

namespace {

std::string read_file(const char* path) {
  std::ifstream in(path, std::ios::binary);
  if (!in) { fprintf(stderr, "cannot read %s\n", path); exit(2); }
  return std::string(std::istreambuf_iterator<char>(in), std::istreambuf_iterator<char>());
}

uint32_t bits_of(float f) { uint32_t u; memcpy(&u, &f, sizeof u); return u; }

int literals(const char* in_path, const char* out_path) {
  const std::string text = read_file(in_path);
  std::vector<unsigned char> accepted;
  std::vector<uint32_t> bits;
  size_t start = 0;
  while (start <= text.size()) {
    size_t end = text.find('\n', start);
    if (end == std::string::npos) end = text.size();
    float v = 0.f;
    const bool ok = parse_field(text.data() + start, text.data() + end, &v);
    accepted.push_back(ok ? 1 : 0);
    bits.push_back(ok ? bits_of(v) : 0u);
    start = end + 1;
  }
  FILE* f = fopen(out_path, "wb");
  if (!f) { fprintf(stderr, "cannot write %s\n", out_path); return 2; }
  fwrite(accepted.data(), 1, accepted.size(), f);
  fwrite(bits.data(), 4, bits.size(), f);
  fclose(f);
  printf("{\"literals\": %zu}\n", accepted.size());
  return 0;
}

// count_newlines_kernel before text_parse.h: a has-zero-byte test used as a per-byte count
int old_newlines(uint32_t word) {
  const uint32_t x = word ^ 0x0a0a0a0au;
  return __builtin_popcount((x - 0x01010101u) & ~x & 0x80808080u);
}

int byte_count(uint32_t word) {
  int c = 0;
  for (int k = 0; k < 4; ++k) c += ((word >> (8 * k)) & 0xffu) == 0x0au;
  return c;
}

int words() {
  const int T = 8;
  struct Part { unsigned long long new_bad = 0, old_bad = 0; uint64_t new_first = ~0ull, old_first = ~0ull; };
  std::vector<Part> parts(T);
  std::vector<std::thread> threads;
  for (int t = 0; t < T; ++t) {
    threads.emplace_back([t, &parts] {
      Part& p = parts[t];
      const uint64_t lo = (uint64_t)t << 29, hi = (uint64_t)(t + 1) << 29;      // 2^32 / 8 words each, in order
      for (uint64_t w64 = lo; w64 < hi; ++w64) {
        const uint32_t w = (uint32_t)w64;
        const int want = byte_count(w);
        if (newlines_in_word(w) != want) { if (!p.new_bad++) p.new_first = w64; }
        if (old_newlines(w) != want) { if (!p.old_bad++) p.old_first = w64; }
      }
    });
  }
  for (auto& th : threads) th.join();
  Part all;
  for (const Part& p : parts) {
    all.new_bad += p.new_bad; all.old_bad += p.old_bad;
    if (p.new_first < all.new_first) all.new_first = p.new_first;
    if (p.old_first < all.old_first) all.old_first = p.old_first;
  }
  printf("{\"words\": %llu, \"new_bad\": %llu, \"new_first_bad\": %lld, \"old_bad\": %llu, \"old_first_bad\": %lld}\n",
         1ull << 32, all.new_bad, all.new_bad ? (long long)all.new_first : -1ll, all.old_bad, all.old_bad ? (long long)all.old_first : -1ll);
  return 0;
}

int libsvm(int mode, const char* in_path, const char* out_path) {
  const std::string text = read_file(in_path);
  FILE* f = fopen(out_path, "w");
  if (!f) { fprintf(stderr, "cannot write %s\n", out_path); return 2; }
  size_t bodies = 0, lines = 0, entries = 0, b0 = 0;
  while (b0 <= text.size()) {
    size_t b1 = text.find('\0', b0);
    if (b1 == std::string::npos) b1 = text.size();
    std::vector<std::pair<size_t, size_t>> rows;                                   // [start, end) of each line
    for (size_t s = b0;;) {
      size_t e = text.find('\n', s);
      if (e == std::string::npos || e > b1) e = b1;
      rows.emplace_back(s, e);
      if (e == b1) break;
      s = e + 1;
    }
    fprintf(f, "body %zu\n", rows.size());
    for (auto& r : rows) {
      std::vector<std::pair<int, uint32_t>> got;
      const bool good = libsvm_line(text.data() + r.first, text.data() + r.second, mode, [&](int idx, float val) {
        got.emplace_back(idx, bits_of(val)); return true;
      });
      fprintf(f, "%d %zu", good ? 1 : 0, got.size());
      for (auto& g : got) fprintf(f, " %d %u", g.first, g.second);
      fputc('\n', f);
      entries += got.size();
    }
    ++bodies; lines += rows.size();
    b0 = b1 + 1;
  }
  fclose(f);
  printf("{\"bodies\": %zu, \"lines\": %zu, \"entries\": %zu}\n", bodies, lines, entries);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "literals" && argc == 4) return literals(argv[2], argv[3]);
  if (cmd == "words" && argc == 2) return words();
  if (cmd == "libsvm" && argc == 5) return libsvm(atoi(argv[2]), argv[3], argv[4]);
  fprintf(stderr, "usage: text_parse_sweep literals IN OUT | words | libsvm MODE IN OUT\n");
  return 2;
}
