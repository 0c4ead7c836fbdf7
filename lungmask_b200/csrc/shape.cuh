// Mesh shape sums and maximum diameters of a label mask (lm_shape_sums_dev, lm_max_diameters_dev; see shape.cu, DESIGN §4.10).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kShapeRows = 257;     // row l = mask == l (row 0 stays zero), row 256 = mask != 0
constexpr int kShapeMoments = 10;   // N, Si, Sj, Sk, Sii, Sjj, Skk, Sij, Sik, Sjk over the array indices (i, j, k)

// Device work buffers of the shape calls, grown on demand and reused across calls.
struct ShapeWork {
  void* d = nullptr;     // the sums; the line tables, candidates, plane histograms and squared diameters
  size_t d_bytes = 0;
  void* f = nullptr;     // the candidates of each diameter family, bucketed by plane, and the bucket offsets
  size_t f_bytes = 0;
  int reserve(size_t bytes, size_t f_bytes_needed);
  void release();
};

// One pass over the (n0,n1,n2) uint8 mask for all rows.  Marching-cube configurations on the mask padded with one voxel
// of outside: counts [257][256] the cubes of each configuration, possum [257][256][3] the sum of their lowest corners p
// (array axes, -1..n_k-1); moments [257][10].  All int64, host memory.  Synchronises `st`.
int shape_sums(ShapeWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int64_t* counts, int64_t* possum, int64_t* moments,
               int num_sms, cudaStream_t st, int64_t* launches);

// The squared maximum distances d2 [4] (host: 3-D, equal axis-0, equal axis-1, equal axis-2 coordinate) between the mesh
// vertices of `row` (1..255: mask == row, 256: mask != 0), spacing s0, s1, s2 per array axis.  0 without vertices.
// Synchronises `st`.
int max_diameters(ShapeWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const double* spacing, double* d2,
                  int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
