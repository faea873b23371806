// rng.h -- the counter-based RNG of subsample and colsample_*, shared by the host, the device and the oracle
// (oracle/gbt_oracle.c): splitmix64 on (seed, stream, index), 24 bits of the hash as a uniform draw in [0, 1).
// The streams are listed at booster.cu subset_mask.
#pragma once

namespace b200 {

__host__ __device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ULL; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL; return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ float rng_uniform(unsigned seed, unsigned long long stream, unsigned long long idx) {
  const unsigned long long h = splitmix64(splitmix64(((unsigned long long)seed << 32) ^ stream) ^ idx);
  return (float)(h >> 40) * (1.0f / 16777216.0f);
}
// subsample's row draw of boosting round `iter`: row `row` (the rank's row offset added) is in the round's sample
__host__ __device__ __forceinline__ bool row_sampled(unsigned seed, unsigned long long iter, unsigned long long row, float subsample) {
  return !(subsample < 1.0f) || rng_uniform(seed, 0x2000ull + iter, row) < subsample;
}

}  // namespace b200
