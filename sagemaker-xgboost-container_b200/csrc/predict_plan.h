// predict_plan.h -- host-side plan of the predictor (no CUDA calls): which kernel runs, how the trees of [tree_begin,
// tree_end) are cut into shared-memory chunks, and the rows and threads of each chunk's CTAs.  launch_predict (misc.cu)
// executes the plan and decides nothing itself; tests/helpers/predict_plan_sweep.cc checks it over a sweep of shapes.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

constexpr size_t kPredictSmem = 220 * 1024;          // dynamic shared memory of a tiled CTA
constexpr size_t kPredictNodeBudget = 96 * 1024;     // packed nodes per chunk (8 B each), at most
constexpr size_t kPredictMinNodeRoom = 64 * 1024;    // rows wider than leave this much beside a 32-row tile: thread-per-row
constexpr int64_t kPredictMaxTreeNodes = 65534;      // 16-bit child index, 0xffff marks a leaf
constexpr int kPredictMaxPitch = 32767;              // 15-bit feature index
constexpr int kPredictMinRows = 32;
constexpr int kPredictMaxRows = 1024;

struct PredictChunk {
  int tree_lo, tree_hi;     // trees [tree_lo, tree_hi) staged together
  size_t node_bytes;        // 8 B per node
  size_t head;              // the chunk's node offsets (16 B aligned) + node_bytes
  int rows, threads;        // rows per tile (a multiple of 32, <= threads), CTA size
  size_t smem;              // head + rows * pitch * 4
};

enum class PredictKernel { kTiled, kThreadPerRow };

struct PredictPlan {
  PredictKernel kernel = PredictKernel::kThreadPerRow;
  const char* reason = "";  // why thread-per-row ("" for the tiled kernel)
  int pitch = 0;            // floats (bins: 4-byte words of bin codes) per staged row (odd)
  bool bins = false;        // the bin predictor (predict_bins.cu) runs the plan
  std::vector<PredictChunk> chunks;
};

// bytes in front of a chunk's row tile: the node offsets of nt trees, 16 B aligned, then the packed nodes
inline size_t predict_chunk_head(int nt, size_t node_bytes) { return (((size_t)(nt + 1) * 4 + 15) & ~(size_t)15) + node_bytes; }

// greedy chunks of [tree_begin, tree_end) for staged rows of row_bytes each: add trees while the nodes stay within the budget
// AND a 32-row tile still fits beside them.  False (reason set) when a tree does not fit.
inline bool plan_predict_chunks(PredictPlan& p, const int64_t* tree_offset, int tree_begin, int tree_end, size_t row_bytes) {
  const size_t tile_min = row_bytes * kPredictMinRows;
  int lo = tree_begin;
  while (lo < tree_end) {
    int hi = lo; size_t bytes = 0;
    while (hi < tree_end) {
      const int64_t nn = tree_offset[hi + 1] - tree_offset[hi];
      if (nn > kPredictMaxTreeNodes) { p.chunks.clear(); p.reason = "tree too large"; return false; }
      const size_t nb = bytes + (size_t)nn * 8;
      const bool fits = nb <= kPredictNodeBudget && predict_chunk_head(hi + 1 - lo, nb) + tile_min <= kPredictSmem;
      if (!fits) {
        if (hi == lo) { p.chunks.clear(); p.reason = "tree too large"; return false; }
        break;
      }
      bytes = nb; ++hi;
    }
    PredictChunk c;
    c.tree_lo = lo; c.tree_hi = hi; c.node_bytes = bytes; c.head = predict_chunk_head(hi - lo, bytes);
    int rows = (int)((kPredictSmem - c.head) / row_bytes);
    rows = rows > kPredictMaxRows ? kPredictMaxRows : (rows / 32) * 32;
    c.threads = rows >= 1024 ? 1024 : (rows >= 512 ? 512 : 256);
    c.rows = rows > c.threads ? c.threads : rows;    // one row per thread and tile
    c.smem = c.head + (size_t)c.rows * row_bytes;
    p.chunks.push_back(c);
    lo = hi;
  }
  p.kernel = PredictKernel::kTiled;
  return true;
}

// tree_offset: node offset of tree t at [t], its end at [t + 1] (per-tree slots, not necessarily contiguous).
// F: columns of the matrix; model_F: features of the model (splits read f < model_F); legacy: force thread-per-row.
inline PredictPlan plan_predict(const int64_t* tree_offset, int tree_begin, int tree_end, int F, int model_F,
                                bool children_adjacent, bool legacy) {
  PredictPlan p;
  p.pitch = F | 1;                                   // odd pitch: threads of a warp (rows) hit different banks for the same feature
  const size_t row_bytes = (size_t)p.pitch * 4;
  if (legacy) { p.reason = "B200XGB_PREDICT_LEGACY"; return p; }
  if (tree_offset == nullptr) { p.reason = "no host tree offsets"; return p; }
  if (!children_adjacent) { p.reason = "children not adjacent"; return p; }
  // a staged row holds F floats: a feature f >= F would read the pad column or the next row, so narrower matrices read
  // their missing columns in the thread-per-row kernel, which takes them as NaN
  if (F < model_F) { p.reason = "matrix narrower than the model"; return p; }
  if (F > kPredictMaxPitch || row_bytes * kPredictMinRows + kPredictMinNodeRoom > kPredictSmem) { p.reason = "rows too wide"; return p; }
  plan_predict_chunks(p, tree_offset, tree_begin, tree_end, row_bytes);
  return p;
}

// The bin predictor's plan (predict_bins.cu): a staged row is the row's bin codes, row_bytes = ngroups * 32 + tw, held in an
// odd number of 4-byte words.  Splits on features the matrix lacks are resolved before the launch (their default direction),
// so a narrower matrix tiles too.
inline PredictPlan plan_predict_bins(const int64_t* tree_offset, int tree_begin, int tree_end, int row_bytes, bool children_adjacent, bool legacy) {
  PredictPlan p;
  p.bins = true;
  p.pitch = ((row_bytes + 3) / 4) | 1;               // words per staged row, odd: a warp's rows hit different banks
  if (legacy) { p.reason = "B200XGB_PREDICT_LEGACY"; return p; }
  if (tree_offset == nullptr) { p.reason = "no host tree offsets"; return p; }
  if (!children_adjacent) { p.reason = "children not adjacent"; return p; }
  if ((size_t)p.pitch * 4 * kPredictMinRows + kPredictMinNodeRoom > kPredictSmem) { p.reason = "rows too wide"; return p; }
  plan_predict_chunks(p, tree_offset, tree_begin, tree_end, (size_t)p.pitch * 4);
  return p;
}

inline std::string predict_plan_json(const PredictPlan& p, int tree_begin, int tree_end, bool has_nan) {
  std::string s = "{\"kernel\":\"";
  if (p.bins) s += p.kernel == PredictKernel::kTiled ? "predict_bins_tiled_kernel" : "predict_bins_kernel";
  else s += p.kernel == PredictKernel::kTiled ? "predict_tiled_kernel" : "predict_kernel";
  s += "\",\"reason\":\""; s += p.reason;
  s += "\",\"has_nan\":"; s += has_nan ? "true" : "false";
  s += ",\"tree_begin\":" + std::to_string(tree_begin) + ",\"tree_end\":" + std::to_string(tree_end);
  s += ",\"pitch\":" + std::to_string(p.pitch) + ",\"chunks\":[";
  for (size_t i = 0; i < p.chunks.size(); ++i) {
    const PredictChunk& c = p.chunks[i];
    if (i) s += ",";
    s += "{\"begin\":" + std::to_string(c.tree_lo) + ",\"end\":" + std::to_string(c.tree_hi) + ",\"node_bytes\":" + std::to_string(c.node_bytes) +
         ",\"rows\":" + std::to_string(c.rows) + ",\"threads\":" + std::to_string(c.threads) + ",\"smem\":" + std::to_string(c.smem) + "}";
  }
  return s + "]}";
}

}  // namespace b200
