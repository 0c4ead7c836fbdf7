// Voxel-based GLCM feature maps of one row of a level map (lm_glcm_maps_dev; see glcm_maps.cu, DESIGN §4.16).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kGlcmMapsFeatures = 22;   // the bits of feature_bits, in texture.GLCM_FEATURES order
constexpr int kGlcmMapsMaxRadius = 3;
constexpr int kGlcmMapsRange = -44;     // a level above n_levels in a window (internal)

// N_max of a radius: twice the pairs of direction (0,0,1) in a full (2r+1)^3 window.
constexpr int glcm_maps_max_n(int radius) { return 2 * (2 * radius + 1) * (2 * radius + 1) * (2 * radius); }

// The scalars of one call, as the C ABI takes them (checked by the caller).
struct GlcmMapsArgs {
  int row;              // 1..255: mask == row; 256: mask > 0
  int radius;           // 1..3
  int n_levels;         // 1..255
  double init_value;
  unsigned bits;        // the requested features, bit k = GLCM_FEATURES[k]
  const double* table;  // device entropy table, N_max (N_max + 1) / 2 entries
};

// Device work buffer: the error flag.
struct GlcmMapsWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// Writes popcount(bits) float64 (n0,n1,n2) planes to d_out (plane j the j-th requested feature).  -> 0,
// kGlcmMapsRange, or a cudaError_t.  Synchronises `st`.
int glcm_maps(GlcmMapsWork& w, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2,
              const GlcmMapsArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
