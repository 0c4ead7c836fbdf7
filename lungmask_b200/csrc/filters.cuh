// PyRadiomics' elementwise image types (Square, SquareRoot, Logarithm, Exponential) and its Gradient image type, one
// float64 image per call, with the range pass that supplies their scalars (lm_image_range_dev, lm_image_filter_dev,
// lm_gradient_dev; see filters.cu, DESIGN §4.13).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kFilterRangeBlocks = 1024;   // the most blocks of the range pass, so its partials fit FilterWork

// Device work buffer of the filter calls: the non-finite flag and the range pass's per-block partials
// (min, max, non-finite) as doubles.
struct FilterWork {
  int* d_flag = nullptr;
  double* d_partial = nullptr;
  int reserve();
  void release();
};

// min and max of the (n) volume `d_vol` (LM_DTYPE_* `dtype`), each voxel converted to float64, into out[0] and out[1]
// (+-inf when every voxel is NaN).  -> 0, LM_ERR_NONFINITE when the volume holds a NaN or +-inf, -1 for an unknown
// dtype, or a cudaError_t.  Synchronises `st`.
int image_range(FilterWork& w, const void* d_vol, int dtype, size_t n, double out[2], int num_sms, cudaStream_t st,
                int64_t* launches);

// One elementwise image type (LM_FILTER_*) of the (n) volume into the float64 (n) `d_out`.  With a table (d_table
// non-NULL, integer dtypes only) out[i] = d_table[x - table_min]; without it the image type's arithmetic with the
// host's scalar `param`.  The caller checks the arguments.  -> 0, LM_ERR_NONFINITE for a NaN or +-inf in the volume,
// LM_ERR_TABLE_RANGE for a voxel outside the table, -1 for an unknown dtype or type, or a cudaError_t.  Synchronises
// `st`.
int image_filter(FilterWork& w, const void* d_vol, int dtype, size_t n, int type, double param, const double* d_table,
                 int64_t table_min, int64_t table_len, double* d_out, int num_sms, cudaStream_t st, int64_t* launches);

// The gradient magnitude of the (n0,n1,n2) volume into the float64 (n0,n1,n2) `d_out`, with inv_xyz = 1 / spacing
// (x = array axis 2, y = 1, z = 0) and clamped neighbours.  -> as image_filter.
int gradient_magnitude(FilterWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, const double inv_xyz[3],
                       double* d_out, cudaStream_t st, int64_t* launches);

}  // namespace lm
