// sampling.h -- sampling_method=gradient_based: minimal-variance row sampling of a tree's gradient pairs
// [UPSTREAM-RECALL: src/tree/gpu_hist/gradient_based_sampler.cu GradientBasedSampler], DESIGN.md "Gradient-based sampling".
// Per column (class) of the round's pairs: rag = sqrtf(g^2 + kGbsLambda h^2), a threshold u with sum_i min(1, rag_i / u) = k
// found by an exact radix descent (no sort, no float scan), then each row kept with probability p = min(1, rag / u) and
// scaled by 1 / p.
#pragma once
#include "engine.h"

namespace b200 {

// The sampler's own regularisation of the hessian in rag; a constant of the sampler, not the tree's reg_lambda
// [UPSTREAM-RECALL: 0.1].  tests/gradient_sampling_reference.py states it once too.
constexpr float kGbsLambda = 0.1f;
// the descent narrows the uint32 bits of rag 8 bits per pass
constexpr int kGbsDigitBits = 8, kGbsBuckets = 1 << kGbsDigitBits, kGbsPasses = 32 / kGbsDigitBits;

// Rows a column of n rows aims to keep: (int64)(float(n) * subsample), computed in float as upstream does, at least 1.
inline long long gbs_target(int64_t n, float subsample) { const long long k = (long long)((float)n * subsample); return k < 1 ? 1 : k; }

// Descent state of one column.  prefix: the rag bits fixed so far; s_lo: rag sum of the rows below the current bucket range
// (the buckets' fixed-point sums, added in double in bucket order), n_hi: rows above it (non-finite rag counts above every
// finite value).  u: the threshold after the last pass.
struct GbsState { unsigned prefix, unused0; double s_lo; long long n_hi; float u; int unused1; };
static_assert(sizeof(GbsState) == 32, "GbsState layout");

struct GbsScratch {
  DevBuf<float> rag;                       // [K][gp_stride]
  DevBuf<unsigned long long> hist;         // [K][2][kGbsBuckets]: row counts, then fixed-point rag sums
  DevBuf<GbsState> st;                     // [K]
};

// The threshold of each of the K columns of gpair ([K][gp_stride], rows [0, n)) into sc->st[k].u, on this rank's rows only.
// u == 0: every row is kept as it is (k >= the rows with rag > 0).  Depends only on the pairs, n and subsample.
void gradient_based_threshold(const float2* gpair, int64_t gp_stride, int64_t n, int K, float subsample, GbsScratch* sc, cudaStream_t s);

// The sample of one tree: per row one draw rng_uniform(seed, stream, r + row_offset), shared by the K columns; column k keeps
// the row when the draw is below p = rag / u_k, as (g / p, h / p) when p < 1.  src may equal dst.  max|g|, max h of what is
// written are folded into absmax (the tree's fixed-point scales).  Reads and writes 8 B per row and column.
struct GbsSampleArgs {
  const float2* src; float2* dst; unsigned* absmax; const GbsState* st;
  int64_t gp_stride, n, row_offset;
  int K; unsigned seed; unsigned long long stream;
};
void launch_gradient_based_sample(const GbsSampleArgs& a, cudaStream_t s);

}  // namespace b200
