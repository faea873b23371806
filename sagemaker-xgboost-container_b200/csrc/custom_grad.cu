// custom_grad.cu -- the caller's gradients as a round's (g, h) pairs (custom_grad.h).  A streaming pass: 8 B read (4 B of g,
// 4 B of h at float32) and 8 B written per row and output.
#include "custom_grad.h"
#include "rng.h"

namespace b200 {

static inline unsigned grid_for(int64_t n) { int64_t g = (n + 255) / 256; if (g < 1) g = 1; if (g > engine_num_sms() * 8) g = engine_num_sms() * 8; return (unsigned)g; }

__device__ __forceinline__ float read_grad(const GradArray& a, int64_t r, int k) {
  const int64_t i = r * a.s0 + (int64_t)k * a.s1;
  return a.f64 ? __double2float_rn(static_cast<const double*>(a.data)[i]) : static_cast<const float*>(a.data)[i];
}

__global__ void __launch_bounds__(256) custom_gradient_kernel(CustomGradArgs a) {
  __shared__ float sg[8], sh[8];
  for (int k = 0; k < a.K; ++k) {          // output by output: each folds its own max|g| and max h under per_target
    float mg = 0.f, mh = 0.f;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
      float g = read_grad(a.g, r, k), h = read_grad(a.h, r, k);
      if (!isfinite(g) || !isfinite(h) || h < 0.f) {
        atomicMin(a.bad, (unsigned long long)(r * a.K + k)); *a.bad_flag = 1u;
        g = 0.f; h = 0.f;
      }
      h = __fadd_rn(h, 0.f);               // -0 to +0: the maxima are folded as unsigned bits
      if (!row_sampled(a.seed, a.iter, (unsigned long long)(r + a.row_offset), a.subsample)) { g = 0.f; h = 0.f; }
      a.gpair[(int64_t)k * a.gp_stride + r] = make_float2(g, h);
      mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
    if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
    __syncthreads();
    if (threadIdx.x == 0 && a.absmax) {
      for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
      unsigned* am = a.absmax + (a.per_target ? 2 * k : 0);
      atomicMax(am, __float_as_uint(mg)); atomicMax(am + 1, __float_as_uint(mh));
    }
    __syncthreads();
  }
}

void launch_custom_gradient(const CustomGradArgs& a, cudaStream_t s) {
  if (a.n == 0) return;
  custom_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
