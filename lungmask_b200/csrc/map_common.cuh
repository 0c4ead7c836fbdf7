// Device helpers shared by the voxel-based texture map kernels (glcm_maps.cu, texture_maps.cu).
#pragma once
#include <stdint.h>

namespace lm {
namespace maps {

typedef unsigned __int128 u128;

// The correctly rounded float64 of a 128-bit integer: the top 64 significant bits with every shifted-out bit ORed into
// bit 0 (a sticky bit below the rounding position), rounded to nearest even, scaled by 2^s exactly.
__device__ __forceinline__ double cvt_u128(u128 m) {
  const unsigned long long hi = (unsigned long long)(m >> 64), lo = (unsigned long long)m;
  if (!hi) return __ull2double_rn(lo);
  const int s = 64 - __clzll((long long)hi);
  unsigned long long top = (unsigned long long)(m >> s);
  if (s == 64 ? lo : (lo & ((1ull << s) - 1))) top |= 1ull;
  return __dmul_rn(__ull2double_rn(top), __longlong_as_double((long long)(1023 + s) << 52));
}

// The offset (dz, dy, dx) of direction d, in texture.OFFSETS order.
__device__ __forceinline__ void offset(int d, int& dz, int& dy, int& dx) {
  if (d < 4) {
    dz = 0;
    dy = d == 0 ? 0 : 1;
    dx = d == 0 ? 1 : d - 2;
  } else {
    dz = 1;
    dy = (d - 4) / 3 - 1;
    dx = (d - 4) % 3 - 1;
  }
}

template <typename T>
__device__ __forceinline__ void insertion_sort(T* v, int n) {
  for (int i = 1; i < n; ++i) {
    const T k = v[i];
    int j = i - 1;
    while (j >= 0 && v[j] > k) {
      v[j + 1] = v[j];
      --j;
    }
    v[j + 1] = k;
  }
}

}  // namespace maps
}  // namespace lm
