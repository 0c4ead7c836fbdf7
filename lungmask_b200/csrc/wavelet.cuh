// Stationary (undecimated) one-level wavelet decomposition of a volume, one band per call (lm_wavelet_dev; see
// wavelet.cu, DESIGN §4.12).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kWaveletBands = 8;   // band = 4 h_x + 2 h_y + h_z, h = 1 for the high-pass filter along that axis

// The filter length of an LM_WAVELET_* code: 6 (coif1), 2 (haar), 0 for an unknown code.
int wavelet_taps(int wavelet);

// Device work buffer of the wavelet call: the non-finite flag.
struct WaveletWork {
  int* d_flag = nullptr;
  int reserve();
  void release();
};

// Band `band` of the (n0,n1,n2) volume `d_vol` (LM_DTYPE_* `dtype`) into the float64 (n0,n1,n2) `d_out`: the x pass (axis
// 2), the y pass (axis 1) and the z pass (axis 0), each out[o] = sum_j f[j] in[(o + F/2 - j) mod N'] with an odd axis
// wrapped to N' = N + 1 (index N holds index 0), every product and sum rounded to float64.  The caller checks the
// arguments (every padded extent at least F, fewer than 2^32 voxels).  -> 0, LM_ERR_NONFINITE when the volume holds a
// NaN or +-inf (d_out is then not a band), -1 for an unknown dtype or wavelet, or a cudaError_t.  Synchronises `st`.
int wavelet_band(WaveletWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, int wavelet, int band, double* d_out,
                 cudaStream_t st, int64_t* launches);

}  // namespace lm
