// Voxel-based GLSZM, GLRLM, GLDM and NGTDM feature maps of one row of a level map (lm_texture_maps_dev; see
// texture_maps.cu, DESIGN §4.17).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

// Class codes (LM_TEXMAP_*) and their feature counts, in texture.*_FEATURES order.
constexpr int kTexMapsGlszm = 1, kTexMapsGlrlm = 2, kTexMapsGldm = 3, kTexMapsNgtdm = 4;
__host__ __device__ constexpr int texture_maps_features(int cls) {
  return cls == kTexMapsGlszm || cls == kTexMapsGlrlm ? 16 : cls == kTexMapsGldm ? 14 : cls == kTexMapsNgtdm ? 5 : 0;
}
constexpr int kTexMapsMaxRadius = 3;
constexpr int kTexMapsRange = -45;   // a level above n_levels in a window (internal)

// The scalars of one call, as the C ABI takes them (checked by the caller).
struct TextureMapsArgs {
  int row;              // 1..255: mask == row; 256: mask > 0
  int radius;           // 1..3
  int n_levels;         // 1..255
  int cls;              // kTexMaps*
  int alpha;            // GLDM: neighbours within alpha levels count, >= 0
  double init_value;
  unsigned bits;        // the requested features of the class, bit k = its k-th feature
  const double* table;  // device entropy table, K (K + 1) / 2 entries, K = (2 radius + 1)^3
};

// Device work buffer: the error flag.
struct TextureMapsWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// Writes popcount(bits) float64 (n0,n1,n2) planes to d_out (plane j the j-th requested feature).  -> 0,
// kTexMapsRange, or a cudaError_t.  Synchronises `st`.
int texture_maps(TextureMapsWork& w, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2,
                 const TextureMapsArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
