// Sweep of the predictor's host-side plan (csrc/predict_plan.h), compiled with g++ by tests/test_predict_plan.py.
//
// For every shape of the sweep it checks the invariants of a plan the tiled kernel can run, and compares the plan with the
// arithmetic of the earlier launch_predict (parent_plan below, kept here to show what changed): where that plan was sound
// the new one must be identical.  Prints one JSON object: the counts, the first violations, the config-5 plan and where
// the earlier arithmetic produced a zero-row tile or tiled a matrix narrower than the model.
#include <algorithm>
#include <cstdio>
#include <map>
#include <random>
#include <string>
#include <vector>

#include "predict_plan.h"

using namespace b200;

namespace {

struct OldChunk { int lo, hi, rows, threads; size_t smem; };
struct OldPlan { bool tiled = false; std::vector<OldChunk> chunks; };

// launch_predict's plan before predict_plan.h: 96 KB chunks, a width gate that assumed 64 KB of nodes, no matrix width check
OldPlan parent_plan(const int64_t* off, int b, int e, int F, bool adjacent, bool legacy) {
  OldPlan p;
  const bool ok = !legacy && off != nullptr && F <= 32767 && adjacent;
  const int pitch = F | 1;
  const size_t kSmem = 220 * 1024;
  if (!(ok && (size_t)pitch * 4 * 32 + 64 * 1024 <= kSmem)) return p;
  const size_t node_budget = 96 * 1024;
  int lo = b; bool fits = true;
  std::vector<std::pair<int, int>> chunks;
  while (lo < e) {
    int hi = lo; size_t bytes = 0;
    while (hi < e) {
      const int64_t nn = off[hi + 1] - off[hi];
      if (nn > 65534) { fits = false; break; }
      if (bytes + (size_t)nn * 8 > node_budget && hi > lo) break;
      if ((size_t)nn * 8 > node_budget) { fits = false; break; }
      bytes += (size_t)nn * 8; ++hi;
    }
    if (!fits) break;
    chunks.emplace_back(lo, hi); lo = hi;
  }
  if (!fits) return p;
  p.tiled = true;
  for (auto& ch : chunks) {
    size_t node_bytes = 0;
    for (int t = ch.first; t < ch.second; ++t) node_bytes += (size_t)(off[t + 1] - off[t]) * 8;
    const size_t head = (((size_t)(ch.second - ch.first + 1) * 4 + 15) & ~(size_t)15) + node_bytes;
    int rows = (int)((kSmem - head) / ((size_t)pitch * 4));
    rows = rows > 1024 ? 1024 : (rows / 32) * 32;
    const int threads = rows >= 1024 ? 1024 : (rows >= 512 ? 512 : 256);
    if (rows > threads) rows = threads;
    p.chunks.push_back({ch.first, ch.second, rows, threads, head + (size_t)rows * pitch * 4});
  }
  return p;
}

struct Stats {
  long plans = 0, tiled = 0, per_row = 0, multi_chunk = 0, min_rows_chunks = 0, compared = 0, changed_where_sound = 0;
  long parent_zero_rows = 0, parent_narrow_tiled = 0;
  std::vector<std::string> violations;
  std::map<std::string, long> reasons;
  std::map<std::string, std::pair<int, int>> zero_row_f;       // label -> [min F, max F] where the parent plan had 0 rows
  void fail(const std::string& what) { if (violations.size() < 20) violations.push_back(what); else violations.back() = "... more"; }
};

std::string where(int F, int mF, int b, int e, bool adj, bool legacy) {
  char s[160];
  snprintf(s, sizeof s, "F=%d model_F=%d trees=[%d,%d) adjacent=%d legacy=%d", F, mF, b, e, (int)adj, (int)legacy);
  return s;
}

// one plan: its invariants, then the comparison with the parent's arithmetic
void check(Stats& st, const std::vector<int64_t>& off, int b, int e, int F, int mF, bool adj, bool legacy, const std::string& label) {
  const PredictPlan p = plan_predict(off.data(), b, e, F, mF, adj, legacy);
  ++st.plans;
  const std::string at = where(F, mF, b, e, adj, legacy);
  const size_t row_bytes = (size_t)(F | 1) * 4;
  auto nodes = [&](int t) { return off[t + 1] - off[t]; };
  if (p.pitch != (F | 1)) st.fail("pitch " + at);
  const bool must_per_row = legacy || !adj || F < mF;
  if (p.kernel == PredictKernel::kTiled) {
    ++st.tiled;
    if (must_per_row) st.fail("tiled although legacy / not adjacent / narrow: " + at);
    if (p.chunks.empty() && b < e) st.fail("no chunks: " + at);
    if (p.chunks.size() > 1) ++st.multi_chunk;
    int next = b;
    for (size_t i = 0; i < p.chunks.size(); ++i) {
      const PredictChunk& c = p.chunks[i];
      if (c.tree_lo != next || c.tree_hi <= c.tree_lo) { st.fail("chunks do not tile the range: " + at); break; }
      size_t bytes = 0;
      for (int t = c.tree_lo; t < c.tree_hi; ++t) {
        if (nodes(t) > kPredictMaxTreeNodes) st.fail("tree over 65534 nodes tiled: " + at);
        bytes += (size_t)nodes(t) * 8;
      }
      const size_t head = (((size_t)(c.tree_hi - c.tree_lo + 1) * 4 + 15) & ~(size_t)15) + bytes;
      if (c.node_bytes != bytes || c.head != head) st.fail("node bytes / head: " + at);
      if (bytes > kPredictNodeBudget) st.fail("chunk over the node budget: " + at);
      if (c.rows < 32 || c.rows > 1024 || c.rows % 32 || c.rows > c.threads) st.fail("rows " + std::to_string(c.rows) + ": " + at);
      if (c.threads != 256 && c.threads != 512 && c.threads != 1024) st.fail("threads: " + at);
      if (c.smem != head + (size_t)c.rows * row_bytes || c.smem > kPredictSmem) st.fail("smem " + std::to_string(c.smem) + ": " + at);
      if (c.rows != c.threads && head + (size_t)(c.rows + 32) * row_bytes <= kPredictSmem) st.fail("tile smaller than the room: " + at);
      if (c.rows == 32) ++st.min_rows_chunks;
      if (i + 1 < p.chunks.size()) {                // greedy: the next tree did not fit into this chunk
        const size_t nb = bytes + (size_t)nodes(c.tree_hi) * 8;
        const size_t h2 = (((size_t)(c.tree_hi - c.tree_lo + 2) * 4 + 15) & ~(size_t)15) + nb;
        if (nb <= kPredictNodeBudget && h2 + 32 * row_bytes <= kPredictSmem) st.fail("chunk cut early: " + at);
      }
      next = c.tree_hi;
    }
    if (next != e) st.fail("chunks end at " + std::to_string(next) + ": " + at);
  } else {
    ++st.per_row; ++st.reasons[p.reason];
    if (!must_per_row) {                             // thread-per-row only when the rows or one tree cannot be tiled
      bool justified = F > kPredictMaxPitch || row_bytes * 32 + kPredictMinNodeRoom > kPredictSmem;
      for (int t = b; t < e && !justified; ++t)
        justified = nodes(t) > kPredictMaxTreeNodes || (size_t)nodes(t) * 8 > kPredictNodeBudget ||
                    16 + (size_t)nodes(t) * 8 + 32 * row_bytes > kPredictSmem;
      if (!justified) st.fail("thread-per-row without cause (" + std::string(p.reason) + "): " + at);
    }
  }
  const OldPlan q = parent_plan(off.data(), b, e, F, adj, legacy);
  if (!q.tiled) return;
  bool zero = false;
  for (auto& c : q.chunks) zero |= c.rows == 0;
  if (zero) {
    ++st.parent_zero_rows;
    auto it = st.zero_row_f.find(label);
    if (it == st.zero_row_f.end()) st.zero_row_f[label] = {F, F};
    else { it->second.first = std::min(it->second.first, F); it->second.second = std::max(it->second.second, F); }
    return;
  }
  if (F < mF) { ++st.parent_narrow_tiled; return; }
  ++st.compared;                                      // the parent plan was sound: nothing may change
  bool same = p.kernel == PredictKernel::kTiled && p.chunks.size() == q.chunks.size();
  for (size_t i = 0; same && i < q.chunks.size(); ++i)
    same = p.chunks[i].tree_lo == q.chunks[i].lo && p.chunks[i].tree_hi == q.chunks[i].hi && p.chunks[i].rows == q.chunks[i].rows &&
           p.chunks[i].threads == q.chunks[i].threads && p.chunks[i].smem == q.chunks[i].smem;
  if (!same) { ++st.changed_where_sound; st.fail("plan changed where the parent's was sound: " + at); }
}

std::vector<int64_t> uniform(int nt, int64_t nodes) {
  std::vector<int64_t> off(nt + 1);
  for (int t = 0; t <= nt; ++t) off[t] = t * nodes;
  return off;
}

int64_t slot(int depth) { return ((((int64_t)1 << (depth + 1)) - 1) + 15) & ~(int64_t)15; }   // round16(2^(d+1) - 1)

// fewest trees of `depth` at which the parent's plan had a zero-row tile (0: none up to 400)
int parent_first_zero(int F, int depth) {
  const std::vector<int64_t> off = uniform(400, slot(depth));
  for (int nt = 1; nt <= 400; ++nt) {
    const OldPlan q = parent_plan(off.data(), 0, nt, F, true, false);
    for (auto& c : q.chunks) if (c.rows == 0) return nt;
  }
  return 0;
}

}  // namespace

int main() {
  Stats st;
  std::vector<int> Fs;
  for (int F = 1; F <= 1400; ++F) Fs.push_back(F);
  for (int F = 1401; F <= 40000; F += 97) Fs.push_back(F);
  for (int F : {2047, 2048, 4095, 4096, 8191, 8192, 16383, 16384, 32766, 32767, 32768, 39999, 40000}) Fs.push_back(F);
  const int counts[] = {1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 191, 192, 193, 255, 256, 257, 383, 384, 385, 400};

  // models of equal trees: a stump, a single split, and the fixed slots of trained trees of depth 1 ... 16
  std::vector<std::pair<std::string, int64_t>> sizes = {{"nodes1", 1}, {"nodes3", 3}};
  for (int d = 1; d <= 16; ++d) sizes.push_back({"depth" + std::to_string(d), slot(d)});
  for (auto& sz : sizes) {
    const std::vector<int64_t> off = uniform(400, sz.second);
    for (int F : Fs)
      for (int nt : counts) {
        check(st, off, 0, nt, F, F, true, false, sz.first);
        if (nt > 2) check(st, off, nt / 3, nt - 1, F, F, true, false, sz.first);     // an iteration range inside the model
        check(st, off, 0, nt, F, F / 2, true, false, sz.first);                        // a matrix wider than the model
        check(st, off, 0, nt, F, F + 1, true, false, sz.first);                        // narrower than the model
        check(st, off, 0, nt, F, F + 3, true, false, sz.first);
        check(st, off, 0, nt, F, F, false, false, sz.first);                           // children not adjacent
        check(st, off, 0, nt, F, F, true, true, sz.first);                             // B200XGB_PREDICT_LEGACY
      }
  }
  // tight node counts (loaded models): random odd sizes of random depths, random ranges
  std::mt19937_64 rng(12345);
  for (int m = 0; m < 300; ++m) {
    const int nt = 1 + (int)(rng() % 400);
    std::vector<int64_t> off(nt + 1, 0);
    for (int t = 0; t < nt; ++t) {
      const int d = 1 + (int)(rng() % 17);
      const int64_t full = ((int64_t)1 << (d + 1)) - 1;
      off[t + 1] = off[t] + 1 + 2 * (int64_t)(rng() % ((full + 1) / 2));
    }
    const int b = (int)(rng() % nt), e = b + 1 + (int)(rng() % (nt - b));
    for (int i = 0; i < 200; ++i) {
      const int F = i < 120 ? 900 + (int)(rng() % 360) : 1 + (int)(rng() % 40000);
      const int mF = (rng() % 4) ? F : F + 1 + (int)(rng() % 5);
      check(st, off, b, e, F, mF, (rng() % 8) != 0, false, "random");
    }
  }

  // BASELINE config 5: 28 features, 50 trees of depth 6
  const std::vector<int64_t> c5 = uniform(50, slot(6));
  const std::string config5 = predict_plan_json(plan_predict(c5.data(), 0, 50, 28, 28, true, false), 0, 50, false);

  printf("{\"plans\":%ld,\"tiled\":%ld,\"per_row\":%ld,\"multi_chunk\":%ld,\"min_rows_chunks\":%ld,\"compared\":%ld,\"changed_where_sound\":%ld,",
         st.plans, st.tiled, st.per_row, st.multi_chunk, st.min_rows_chunks, st.compared, st.changed_where_sound);
  printf("\"parent_zero_rows\":%ld,\"parent_narrow_tiled\":%ld,\"reasons\":{", st.parent_zero_rows, st.parent_narrow_tiled);
  bool first = true;
  for (auto& r : st.reasons) { printf("%s\"%s\":%ld", first ? "" : ",", r.first.c_str(), r.second); first = false; }
  printf("},\"parent_zero_row_f\":{");
  first = true;
  for (auto& z : st.zero_row_f) { printf("%s\"%s\":[%d,%d]", first ? "" : ",", z.first.c_str(), z.second.first, z.second.second); first = false; }
  printf("},\"parent_first_zero_depth6\":{\"1000\":%d,\"1247\":%d},\"config5\":%s,\"violations\":[", parent_first_zero(1000, 6),
         parent_first_zero(1247, 6), config5.c_str());
  for (size_t i = 0; i < st.violations.size(); ++i) printf("%s\"%s\"", i ? "," : "", st.violations[i].c_str());
  printf("]}\n");
  return 0;
}
