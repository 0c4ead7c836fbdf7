// Grey-level texture matrices of one ROI (lm_texture_levels_dev, lm_glcm_dev, lm_glrlm_dev, lm_neighbour_counts_dev,
// lm_glcm_offsets_dev, lm_neighbour_offsets_dev; see texture.cu, DESIGN §4.9 and §4.18).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kGlcmDirections = 13;    // the offsets of the 26-neighbourhood whose first non-zero component is positive
constexpr int kTextureMaxLevels = 255;
constexpr int kNeighbourCells = 27;    // W or c = 0..26 neighbours of the 26-neighbourhood
constexpr int kMaxOffsets = 171;       // the half-space offsets of Chebyshev norm 1..3 (DESIGN §4.18)

// Device work buffers of the texture calls, grown on demand and reused across calls.
struct TextureWork {
  void* d = nullptr;     // the error flag, then the counters of the call: the [13][n_levels (n_levels + 1) / 2] uint32 pair
                         // counts, the [13][n_levels][max(n0,n1,n2)] uint32 run counts, or the uint64 A and uint32 G
                         // and N [n_levels][27] neighbourhood counts
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Errors of texture_levels / glcm / glrlm / neighbour_counts besides a cudaError_t: -1 unknown dtype, kLevelRange a level outside
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

// The run counts P_d(i, k) of the level map for the 13 directions of glcm: counts [13][n_levels][max(n0,n1,n2)] int64
// (host), runs of level i + 1 and length k + 1.  Synchronises `st`.
int glrlm(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, int num_sms,
          cudaStream_t st, int64_t* launches);

// The 26-neighbourhood counts of every ROI voxel v of level i, with W(v) its neighbours in the ROI, S(v) the sum of their
// levels and c(v) those within `alpha` levels of i: dependence G(i, c), ngtdm_counts N(i, W), ngtdm_sums A(i, W) =
// sum |W i - S|, each [n_levels][27] int64 (host).  Synchronises `st`.
int neighbour_counts(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                     int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums, int num_sms, cudaStream_t st,
                     int64_t* launches);

// glcm over a caller's list of n_offsets half-space offsets (int8 [n][3] (dz, dy, dx), host, checked by the caller):
// counts [n][T] int64 (host) in the triangle order of glcm.  The offsets run in groups whose counters fit the shared
// budget of glcm.  Synchronises `st`.
int glcm_offsets(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, const int8_t* offsets,
                 int n_offsets, int64_t* counts, int num_sms, cudaStream_t st, int64_t* launches);

// neighbour_counts over the neighbourhood +-offsets (K = 2 n_offsets neighbours): each output [n_levels][K + 1] int64
// (host).  The counters sit in shared memory while n_levels (K + 1) 16 B fit glcm's budget, in global memory otherwise.
// Synchronises `st`.
int neighbour_offsets(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                      const int8_t* offsets, int n_offsets, int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums,
                      int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
