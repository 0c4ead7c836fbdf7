// PyRadiomics' resampling with the cubic B-spline or nearest-neighbour interpolator: the float64 B-spline coefficient
// volume and the evaluation on an output grid of continuous-index tables (lm_bspline_coefficients_dev, lm_resample_dev;
// see resample.cu, DESIGN §4.19).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

// Device work buffer of the resample calls: the non-finite flag.
struct ResampleWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// The cubic B-spline pole and its filter constants, formed on the host in float64 as written: z = sqrt(3) - 2,
// gain = (1 - z)(1 - 1/z), inv_z = 1/z, anti = z / (z z - 1).
struct BsplinePole {
  double z, gain, inv_z, anti;
};
BsplinePole bspline_pole();

// The float64 B-spline coefficients of the (n0,n1,n2) volume `d_vol` (LM_DTYPE_* `dtype`) into `d_coeff`: a pass along
// x (array axis 2) that also converts the dtype, then y, then z.  The caller checks the arguments.  -> 0,
// LM_ERR_NONFINITE for a NaN or +-inf in the volume, -1 for an unknown dtype, or a cudaError_t.  Synchronises `st`.
int bspline_coefficients(ResampleWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, double* d_coeff,
                         cudaStream_t st, int64_t* launches);

// Samples the (n0,n1,n2) input on the (m0,m1,m2) grid of the float64 tables d_cz [m0], d_cy [m1], d_cx [m2]: the image
// into d_out (the input's dtype) from d_coeff (interpolator LM_RESAMPLE_BSPLINE) or d_vol (LM_RESAMPLE_NEAREST), and the
// mask into the uint8 d_out_mask, in one pass.  The caller checks the arguments.  -> 0, LM_ERR_NONFINITE when a sampled
// coefficient or voxel is a NaN or +-inf, -1 for an unknown dtype, or a cudaError_t.  Synchronises `st`.
int resample_volume(ResampleWork& w, const void* d_vol, int dtype, const double* d_coeff, const uint8_t* d_mask, int n0,
                    int n1, int n2, const double* d_cz, const double* d_cy, const double* d_cx, int m0, int m1, int m2,
                    int interpolator, void* d_out, uint8_t* d_out_mask, cudaStream_t st, int64_t* launches);

}  // namespace lm
