// First-order (histogram) sums of every row of a label mask (lm_first_order_sums_dev, lm_first_order_splits_dev; see
// first_order.cu, DESIGN §4.11).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kFoRows = 257;          // row l = mask == l (row 0 is never a row), row 256 = mask > 0
constexpr int kFoLevels = 256;        // histogram stride: levels 1..255 at their own index, index 0 unused
constexpr int kFoIntSums = 10;        // S1, S2, S3, S4, S_B as (low, high) 64-bit word pairs
constexpr int kFoFloatSums = 5;       // sum e, e^2, e^3, e^4, sum e over the band
constexpr int kFoSplits = 4;          // n_lo, L, n_lo_B, L_B (exact rows); sum |x - mu|, sum_B |x - mu_B| (float rows)
constexpr int64_t kFoExactSpan = (int64_t)1 << 20;   // an exact row's values lie in [base, base + 2^20)
constexpr int kFoSkip = 0, kFoFloat = 1, kFoExact = 2;   // row modes

// Device work buffers of the first-order calls, grown on demand and reused across calls.
struct FirstOrderWork {
  void* d = nullptr;     // the error flag, the slot table, the row parameters and the counters of the call
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Per-row inputs, host arrays indexed 0..256 (row 0 must be kFoSkip).  Pass A reads mode, low, n_levels, base, centre and
// the band; pass B reads mode, base, split / split_band (exact rows), centre / centre_band (float rows) and the band.
struct FirstOrderRows {
  const int* mode;
  const int64_t* low;
  const int* n_levels;
  const int64_t* base;
  const double* centre;
  const double* centre_band;
  const double* band_lo;
  const double* band_hi;
  const int64_t* split;
  const int64_t* split_band;
};

// A value of an exact row outside [base, base + 2^20), or a level outside 1..n_levels, found on the device.
constexpr int kFoRange = -62;

// Pass A over the (n) volume `d_vol` (LM_DTYPE_* `dtype`) and the mask, for every row with a mode: the level histogram
// hist [257][256] int64, and per exact row the 128-bit sums of d^k (d = x - base, k = 1..4) and of d over the band
// int_sums [257][10] (uint64 word pairs), per float row the float64 sums of e^k (e = x - centre) and of e over the band
// float_sums [257][5]; band_count [257] int64.  All host memory.  The caller checks the arguments.  Synchronises `st`.
int first_order_sums(FirstOrderWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, int bin_width,
                     const FirstOrderRows& rows, int64_t* hist, uint64_t* int_sums, int64_t* band_count, double* float_sums,
                     int num_sms, cudaStream_t st, int64_t* launches);

// Pass B: per exact row the count and the sum of d of the voxels with d <= split, and of the band's voxels with
// d <= split_band: below [257][4] int64; per float row sum |x - centre| and the band's sum |x - centre_band|:
// abs_dev [257][2] float64.  Host memory.  Synchronises `st`.
int first_order_splits(FirstOrderWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n,
                       const FirstOrderRows& rows, int64_t* below, double* abs_dev, int num_sms, cudaStream_t st,
                       int64_t* launches);

}  // namespace lm
