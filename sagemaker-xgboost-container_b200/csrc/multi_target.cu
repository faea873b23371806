// multi_target.cu -- multi-target regression (multi_target.h): the gradient pass over T label columns, sibling of misc.cu's
// gradient_kernel as adaptive.cu's quantile_gradient_kernel is, and the element-wise metrics over the n x T elements.  Both
// read the per-element formulas of elementwise.h, so target j computes what gradient_kernel / metric_kernel compute for a
// model trained on label column j alone.  Built with misc.cu's default flags (elementwise.h, transform.h).
#include "elementwise.h"
#include "multi_target.h"
#include "rng.h"

namespace b200 {

static inline unsigned grid_for(int64_t n) { int64_t g = (n + 255) / 256; if (g < 1) g = 1; if (g > engine_num_sms() * 8) g = engine_num_sms() * 8; return (unsigned)g; }

__global__ void __launch_bounds__(256) multi_target_gradient_kernel(MultiGradArgs a) {
  __shared__ float sg[8], sh[8];
  const bool abserr = a.objective == kAbsoluteError, reg_loss = objective_is_reg_loss(a.objective);
  for (int j = 0; j < a.T; ++j) {          // target by target: each folds its own max|g| and max h
    float mg = 0.f, mh = 0.f;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (int64_t)gridDim.x * blockDim.x) {
      const int64_t e = r * a.T + j;
      const float y = a.label[e], m = a.margin ? a.margin[e] : 0.f;
      float w = a.weight ? a.weight[r] : 1.0f, g, h;
      if (abserr) {                        // adaptive.cu abserr_gradient_kernel
        const float diff = __fsub_rn(m, y);
        g = __fmul_rn((float)((diff > 0.f) - (diff < 0.f)), w); h = w;
        if (a.resid) a.resid[j * a.n + r] = __fsub_rn(y, m);
      } else {                             // misc.cu gradient_kernel
        if (reg_loss && y == 1.0f) w *= a.scale_pos_weight;
        elementwise_gradient(a.objective, y, m, a.aux, a.err, &g, &h);
        g *= w; h *= w;
      }
      if (a.subsample < 1.0f && !(rng_uniform(a.seed, 0x2000ull + a.iter, (unsigned long long)(r + a.row_offset)) < a.subsample)) { g = 0.f; h = 0.f; }
      a.gpair[j * a.gp_stride + r] = make_float2(g, h);
      mg = fmaxf(mg, fabsf(g)); mh = fmaxf(mh, h);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o)); }
    if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = mg; sh[threadIdx.x >> 5] = mh; }
    __syncthreads();
    if (threadIdx.x == 0 && a.absmax) {
      for (int w = 1; w < 8; ++w) { mg = fmaxf(mg, sg[w]); mh = fmaxf(mh, sh[w]); }
      unsigned* am = a.absmax + (a.per_target ? 2 * j : 0);
      atomicMax(am, __float_as_uint(mg)); atomicMax(am + 1, __float_as_uint(mh));
    }
    __syncthreads();
  }
}
void launch_multi_target_gradient(const MultiGradArgs& a, cudaStream_t s) {
  B200_CHECK(objective_is_multi_target(a.objective) && a.T >= 1, "multi-target gradient: unsupported objective");
  if (a.n == 0) return;
  multi_target_gradient_kernel<<<grid_for(a.n), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

__global__ void __launch_bounds__(256) multi_target_metric_kernel(MultiMetricArgs a) {
  double s = 0, ws = 0;
  const int64_t total = a.n * a.T;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const float w = a.weight ? a.weight[e / a.T] : 1.0f;
    const float loss = elementwise_loss(a.metric, a.label[e], metric_prediction(a.margin[e], a.is_logistic, a.transform), a.threshold, a.aux);
    s += (double)(loss * w); ws += (double)w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(a.out, s); atomicAdd(a.out + 1, ws); }
}
void launch_multi_target_metric(const MultiMetricArgs& a, cudaStream_t s) {
  if (a.n == 0) return;
  multi_target_metric_kernel<<<grid_for(a.n * a.T), 256, 0, s>>>(a); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

__global__ void __launch_bounds__(256) label_column_kernel(const float* label, int64_t n, int T, int j, float* out) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) out[r] = label[r * T + j];
}
void launch_label_column(const float* label, int64_t n, int T, int j, float* out, cudaStream_t s) {
  if (n == 0) return;
  label_column_kernel<<<grid_for(n), 256, 0, s>>>(label, n, T, j, out); ++g_kernel_launches; CUDA_OK(cudaGetLastError());
}

}  // namespace b200
