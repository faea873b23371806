// auc.cu -- binary ROC-AUC on the device (sort based), checked on hardware against sklearn.metrics.roc_auc_score
// (tests/test_gpu_parity.py::test_auc_matches_sklearn).  Like `aucpr`, `auc` is a metric of the container's HPO list that the
// container does not compute itself (algorithm_mode/train_utils.py:45-76 routes accuracy/f1/rmse/mae... to feval; `auc` and
// `aucpr` stay native).  This file computes binary `auc` on a one-output model; `aucpr` and one-vs-rest `auc` are curve.cu's.
// Definition restated from upstream src/metric/auc.cc (BinaryROCAUC): predictions sorted descending, one trapezoid per
// group of tied predictions, area / (sum_w_pos * sum_w_neg); distributed: sum of local areas / sum of local pos*neg products.
#include <cub/cub.cuh>
#include "engine.h"
#include "misc.h"

namespace b200 {

__global__ void auc_prepare_kernel(const float* margin, int64_t n, int is_logistic, float* keys, int* idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float p = margin[i];
    if (is_logistic) { const float kEps = 1e-16f; float x = fminf(-p, 88.7f); p = 1.0f / (expf(x) + 1.0f + kEps); }
    keys[i] = p; idx[i] = (int)i;
  }
}
__global__ void auc_gather_kernel(const int* idx, const float* skeys, const float* label, const float* weight, int64_t n,
                                  double* wpos, double* wneg, unsigned char* boundary) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = idx[i];
    const double w = weight ? (double)weight[r] : 1.0, y = (double)label[r];
    wpos[i] = w * y; wneg[i] = w * (1.0 - y);
    boundary[i] = (i == n - 1 || skeys[i] != skeys[i + 1]) ? 1 : 0;
  }
}
__global__ void auc_area_kernel(const double* tpb, const double* fpb, const int* m_ptr, double* out) {
  const int m = *m_ptr;
  double acc = 0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
    const double tp0 = j ? tpb[j - 1] : 0.0, fp0 = j ? fpb[j - 1] : 0.0;
    acc += (fpb[j] - fp0) * (tpb[j] + tp0) * 0.5;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc != 0.0) atomicAdd(out, acc);
  if (blockIdx.x == 0 && threadIdx.x == 0 && m > 0) { out[1] = tpb[m - 1]; out[2] = fpb[m - 1]; }
}

// out (device, 3 doubles): [0] += unnormalised area, [1] = sum of positive weight, [2] = sum of negative weight
void compute_auc_device(const float* margin, const float* label, const float* weight, int64_t n, int is_logistic, double* out, cudaStream_t s) {
  CUDA_OK(cudaMemsetAsync(out, 0, 3 * sizeof(double), s));
  if (n == 0) return;
  B200_CHECK(n < (int64_t)0x7fffffff, "auc: too many rows");
  DevBuf<float> keys, skeys; DevBuf<int> idx, sidx, m; DevBuf<double> wpos, wneg, tpb, fpb; DevBuf<unsigned char> boundary, tmp;
  keys.alloc(n); skeys.alloc(n); idx.alloc(n); sidx.alloc(n); m.alloc(1); wpos.alloc(n); wneg.alloc(n); tpb.alloc(n); fpb.alloc(n); boundary.alloc(n);
  const int grid = (int)std::min<int64_t>((n + 255) / 256, engine_num_sms() * 16);
  auc_prepare_kernel<<<grid, 256, 0, s>>>(margin, n, is_logistic, keys.p, idx.p); ++g_kernel_launches;
  size_t need = 0, bytes = 0;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, need, keys.p, skeys.p, idx.p, sidx.p, (int)n, 0, 32, s); bytes = std::max(bytes, need);
  cub::DeviceScan::InclusiveSum(nullptr, need, wpos.p, wpos.p, (int)n, s); bytes = std::max(bytes, need);
  cub::DeviceSelect::Flagged(nullptr, need, wpos.p, boundary.p, tpb.p, m.p, (int)n, s); bytes = std::max(bytes, need);
  tmp.alloc(bytes + 16);
  size_t b = bytes;
  CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(tmp.p, b, keys.p, skeys.p, idx.p, sidx.p, (int)n, 0, 32, s));
  auc_gather_kernel<<<grid, 256, 0, s>>>(sidx.p, skeys.p, label, weight, n, wpos.p, wneg.p, boundary.p); ++g_kernel_launches;
  b = bytes; CUDA_OK(cub::DeviceScan::InclusiveSum(tmp.p, b, wpos.p, wpos.p, (int)n, s));
  b = bytes; CUDA_OK(cub::DeviceScan::InclusiveSum(tmp.p, b, wneg.p, wneg.p, (int)n, s));
  b = bytes; CUDA_OK(cub::DeviceSelect::Flagged(tmp.p, b, wpos.p, boundary.p, tpb.p, m.p, (int)n, s));
  b = bytes; CUDA_OK(cub::DeviceSelect::Flagged(tmp.p, b, wneg.p, boundary.p, fpb.p, m.p, (int)n, s));
  auc_area_kernel<<<grid, 256, 0, s>>>(tpb.p, fpb.p, m.p, out); ++g_kernel_launches;
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(s));        // the temporaries die with this scope
}

}  // namespace b200
