// Reading a uint8 label mask 16 voxels at a time (stats.cu, clusters.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kChunk = 16;          // voxels per thread and step: one 16-byte mask vector

// The 16 labels of a chunk as one vector (a 16-byte load where the mask allows it; 0 past the end).
__device__ __forceinline__ uint4 load_labels(const uint8_t* __restrict__ m, size_t base, size_t n) {
  if (base + kChunk <= n && (reinterpret_cast<uintptr_t>(m) & 15) == 0) return __ldg(reinterpret_cast<const uint4*>(m + base));
  unsigned w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < kChunk; ++k)
    if (base + k < n) w[k >> 2] |= (unsigned)m[base + k] << (8 * (k & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}
// Label k of the chunk, with selects rather than an indexed array (no local memory when the loop is not unrolled).
__device__ __forceinline__ int label_at(const uint4& u, int k) {
  const unsigned w = k < 8 ? (k < 4 ? u.x : u.y) : (k < 12 ? u.z : u.w);
  return (int)((w >> (8 * (k & 3))) & 255u);
}

}  // namespace lm
