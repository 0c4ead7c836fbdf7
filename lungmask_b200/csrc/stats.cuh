// Per-label volume and HU statistics of a (volume, mask) pair (see stats.cu, DESIGN §4.6).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kStatsBins = 4098;   // [under (< -1024), -1024, ..., 3071, over (>= 3072)]: 1-HU bins of floor(value)
constexpr int kStatsRows = 257;    // rows 0..255 = label values, row 256 = the union (mask > 0)

// Where label_stats writes its results (host memory, kStatsRows rows each, see lm_label_stats_dev in the header).
struct LabelStatsOut {
  int64_t* voxels;       // [257]
  int64_t* nan_voxels;   // [257]
  double* moments;       // [257][4]: mean, std (ddof 0), min, max
  double* percentile;    // [257][n_q]
  int64_t* below;        // [257][n_t]: count(value < t)
};

// Device work buffers and host staging of label_stats, grown on demand and reused across calls.
struct LabelStatsWork {
  void* d = nullptr;          // device: counts, slot table, histograms, accumulators, selection targets
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Statistics of `d_vol` (n voxels of element type `dtype`, an LM_DTYPE_* code) per label of `d_mask` (n uint8).  Both on
// the current device.  Enqueues on `st` and synchronises it (three times: after the count pass, after the histogram
// pass and at the end).  q in [0, 100], t in [-1024, 3072]: the caller checks them.  Returns 0, a cudaError_t, or -1 for
// an unknown dtype.  *launches += the kernels launched.
int label_stats(LabelStatsWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, const double* q, int n_q,
                const int* t, int n_t, const LabelStatsOut& out, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
