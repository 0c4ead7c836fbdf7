// Voxel-based first-order feature maps of one row of a label mask (lm_first_order_maps_dev; see first_order_maps.cu,
// DESIGN §4.15).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kFomFeatures = 18;        // the bits of feature_bits, in first_order.FIRST_ORDER_FEATURES order
constexpr int kFomMaxRadius = 3;
constexpr int kFomRange = -43;          // a candidate outside its exact span or a level outside 1..n_levels (internal)

// The scalars of one call, as the C ABI takes them (checked by the caller).
struct FomArgs {
  int row;             // 1..255: mask == row; 256: mask > 0
  int radius;          // 1..3
  int masked;          // candidates W(c) & ROI (1) or the non-NaN voxels of W(c) (0)
  int bin_width;
  int n_levels;
  int exact;           // integer dtypes only
  long long low, base, shift;
  double voxel_volume, init_value;
  unsigned bits;       // the requested features, bit k = FIRST_ORDER_FEATURES[k]
  const double* table; // device entropy table, (2r+1)^3 ((2r+1)^3 + 1) / 2 entries
};

// Device work buffer: the error flag.
struct FomWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// Writes popcount(bits) float64 (n0,n1,n2) planes to d_out (plane j the j-th requested feature).  -> 0,
// LM_ERR_NONFINITE for a +-inf candidate, kFomRange, -1 for an unknown dtype, or a cudaError_t.  Synchronises `st`.
int first_order_maps(FomWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                     const FomArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
