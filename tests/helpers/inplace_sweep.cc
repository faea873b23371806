// The host half of csrc/inplace.h over a sweep, without a GPU (tests/test_inplace_predict_host.py): typestr parsing, and the
// row chunks of host inputs.  Every dense plan must cover [0, n) with chunks that fit the staging buffer and honour the debug
// cap; every CSR plan likewise, refusing only rows that alone exceed the buffer.  Prints one JSON object.
#include <cstdio>
#include <random>
#include <string>
#include <vector>
#include "inplace.h"

using namespace b200;

int main() {
  long long violations = 0, dense_plans = 0, csr_plans = 0, multi_chunk = 0, refused_rows = 0;
  std::string types;
  for (const char* ts : {"<f4", "<f8", "<f2", "|i1", "<i2", "<i4", "<i8", "|u1", "<u2", "<u4", "<u8", "|b1", "<c8", "<c16", "|O", "<M8[ns]", "<m8[s]", ">f4", "<V8"}) {
    std::string why; const int t = in_type_of(ts, &why);
    char buf[160]; snprintf(buf, sizeof buf, "%s\"%s\":[%d,%d,\"%s\"]", types.empty() ? "" : ",", ts, t, t >= 0 ? in_itemsize(t) : 0, why.c_str());
    types += buf;
  }
  const size_t caps[] = {64, 1000, 4096, kInplaceStageBytes};
  for (size_t cap : caps)
    for (int64_t n : {0LL, 1LL, 2LL, 7LL, 63LL, 64LL, 65LL, 1000LL, 65536LL, 10000000LL})
      for (int64_t rb : {1LL, 4LL, 8LL, 28LL, 112LL, 224LL, 800LL, 4096LL})
        for (int64_t dbg : {0LL, 1LL, 3LL, 64LL}) {
          if (!inplace_row_fits(rb, cap)) { ++refused_rows; continue; }
          ++dense_plans;
          const int64_t rows = inplace_chunk_rows(n, rb, cap, dbg);
          if (rows < 1 || (n > 0 && rows > n) || (size_t)(rows * rb) > cap || (dbg > 0 && rows > dbg)) ++violations;
          if (n > rows) ++multi_chunk;
        }
  std::mt19937_64 rng(7);
  for (int trial = 0; trial < 3000; ++trial) {
    const int64_t n = (int64_t)(rng() % 300);
    std::vector<int64_t> ip(n + 1, 0);
    for (int64_t r = 0; r < n; ++r) ip[r + 1] = ip[r] + (int64_t)(rng() % 4 == 0 ? rng() % 200 : rng() % 8);
    const size_t cap = caps[rng() % 3];
    const int64_t dbg = (int64_t)(rng() % 3 == 0 ? rng() % 5 : 0);
    int64_t r0 = 0; bool refused = false;
    while (r0 < n) {
      const int64_t r1 = inplace_csr_chunk_end(ip.data(), n, r0, cap, dbg);
      if (r1 == r0) {
        if (inplace_csr_bytes(1, ip[r0 + 1] - ip[r0]) <= cap) ++violations;
        refused = true; break;
      }
      if (inplace_csr_bytes(r1 - r0, ip[r1] - ip[r0]) > cap || (dbg > 0 && r1 - r0 > dbg)) ++violations;
      // maximal: one more row would not fit (or the debug cap / the end stops it)
      if (r1 < n && !(dbg > 0 && r1 - r0 == dbg) && inplace_csr_bytes(r1 + 1 - r0, ip[r1 + 1] - ip[r0]) <= cap) ++violations;
      if (r1 < n) ++multi_chunk;
      r0 = r1;
    }
    if (refused) ++refused_rows;
    ++csr_plans;
  }
  printf("{\"violations\":%lld,\"dense_plans\":%lld,\"csr_plans\":%lld,\"multi_chunk\":%lld,\"refused\":%lld,\"types\":{%s}}\n",
         violations, dense_plans, csr_plans, multi_chunk, refused_rows, types.c_str());
  return 0;
}
