// Pieces of scikit-learn's KMeans that the per-image clustering (segment.cu) and the data-set clustering (cluster.cu)
// share: the counter-based random generator that replaces numpy's global RNG, and the number of local trials of the
// greedy k-means++ seeding (sklearn _kmeans_plusplus: 2 + floor(ln k)).
#pragma once
#include <math.h>
#include <stdint.h>

namespace dss {

__device__ __forceinline__ uint32_t seg_hash(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t x = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du;
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}
// uniform in [0, 1) with 24 random bits, keyed by (seed, stream key, counter)
__device__ __forceinline__ double seg_uniform(uint32_t seed, uint32_t img, uint32_t ctr) {
  return (double)(seg_hash(seed, img, ctr) >> 8) * (1.0 / 16777216.0);
}

__host__ __device__ __forceinline__ int kmeans_local_trials(int k) { return 2 + (int)log((double)k); }

}  // namespace dss
