// PyRadiomics' LoG image type: ITK's LaplacianRecursiveGaussianImageFilter with NormalizeAcrossScale, as nine separable
// 4th-order recursive line passes in float64 (lm_laplacian_of_gaussian_dev; see laplacian.cu, DESIGN §4.20).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

// Device work buffer of the LoG call: the non-finite flag.
struct LogWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// The coefficients of one recursive line filter (lungmask_b200.laplacian.LineCoefficients): the causal numerator
// N0..N3, the anticausal numerator M1..M4, the shared denominator D1..D4 and the boundary terms BN1..BN4, BM1..BM4.
struct LogLine {
  double n[4], m[4], d[4], bn[4], bm[4];
};

// The line filter of order 0 (smoothing) or 2 (second derivative times sd^2) for sd = sigma / spacing samples, formed on
// the host in float64 with the operations of lungmask_b200.laplacian.coefficients in the same order.
LogLine log_line_coefficients(double sd, int order);

// The LoG of the (n0,n1,n2) volume `d_vol` (LM_DTYPE_* `dtype`) into the float64 d_out: for d = x, y, z the order-0
// filter `smooth[a]` along the two other axes a (in x, y, z order) and the order-2 filter `deriv[d]` along d, the terms
// summed from +0.0.  d_work0 and d_work1 are float64 volumes of the input's size.  The caller checks the arguments
// (every extent >= 4, no overlaps).  -> 0, LM_ERR_NONFINITE for a NaN or +-inf in the volume, -1 for an unknown dtype,
// or a cudaError_t.  Synchronises `st`.
int laplacian_of_gaussian(LogWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, const LogLine smooth[3],
                          const LogLine deriv[3], double* d_work0, double* d_work1, double* d_out, cudaStream_t st,
                          int64_t* launches);

}  // namespace lm
