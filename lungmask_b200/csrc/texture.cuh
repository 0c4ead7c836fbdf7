// Grey-level texture matrices of one ROI (lm_texture_levels_dev, lm_glcm_dev; see texture.cu, DESIGN §4.9).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kGlcmDirections = 13;    // the offsets of the 26-neighbourhood whose first non-zero component is positive
constexpr int kTextureMaxLevels = 255;

// Device work buffers of the texture calls, grown on demand and reused across calls.
struct TextureWork {
  void* d = nullptr;     // the error flag and the [13][n_levels (n_levels + 1) / 2] uint32 pair counts
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Errors of texture_levels / glcm besides a cudaError_t: -1 unknown dtype, kLevelRange a level outside
// 1..n_levels, kLevelNonFinite a non-finite value in the ROI (both found on the device; the map is then incomplete).
constexpr int kLevelRange = -60;
constexpr int kLevelNonFinite = -61;

// The uint8 level map of `row` (1..255: mask == row, 256: mask > 0) of the (n) volume `d_vol` (LM_DTYPE_* `dtype`) and
// the mask: level(x) = floor((floor(x) - low) / bin_width) + 1 in int64 under the row where x is not NaN, 0 elsewhere.
// d_levels: n bytes, 16-byte aligned.  The caller checks the arguments.  Synchronises `st`.
int texture_levels(TextureWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, int row, int64_t low,
                   int bin_width, int n_levels, uint8_t* d_levels, int num_sms, cudaStream_t st, int64_t* launches);

// The unordered pair counts U_d(i <= j) of the (n0,n1,n2) level map for the 13 directions: counts [13][T] int64 (host),
// T = n_levels (n_levels + 1) / 2, (i, j) in row-major upper-triangle order.  Synchronises `st`.
int glcm(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, int num_sms,
         cudaStream_t st, int64_t* launches);

}  // namespace lm
