// custom_grad.h -- custom objectives (DESIGN.md "Custom objectives"): the caller's gradient and hessian arrays turned into a
// round's (g, h) pairs on the device (custom_grad.cu), in place of the objective's gradient pass.
#pragma once
#include "engine.h"

namespace b200 {

// One of the caller's (n, K) arrays on the engine's device: element (r, k) is at data + r * s0 + k * s1 (strides in elements,
// either sign), float32 (f64 == 0) or float64 (f64 == 1, rounded to float32 when read).
struct GradArray { const void* data; int64_t s0, s1; int f64; };

// Pair (r, k) is (g[r][k], h[r][k]) into gpair[k * gp_stride + r], or (0, 0) when row r is outside round `iter`'s subsample
// draw (rng.h row_sampled, as gradient_kernel draws it).  absmax (may be nullptr): max|g| and max h of the written pairs into
// [0] and [1], or with per_target each output k's into [2 k] and [2 k + 1].  Every element is checked, sampled or not: a
// non-finite g or h or an h < 0 sets *bad_flag = 1 and atomicMin's r * K + k into *bad (the caller sets it to ~0 first).
struct CustomGradArgs {
  GradArray g, h;
  float2* gpair; int64_t gp_stride; unsigned* absmax; int per_target;
  unsigned long long* bad; unsigned* bad_flag;
  int64_t n, row_offset; int K;
  float subsample; unsigned seed; unsigned long long iter;
};
void launch_custom_gradient(const CustomGradArgs& a, cudaStream_t s);

}  // namespace b200
