// First-order (histogram) sums of every row of a label mask (lm_first_order_sums_dev, lm_first_order_splits_dev,
// DESIGN §4.11).
//
// Both passes run once over the (volume, mask) pair for all rows, grid-stride over 16-voxel chunks (one 16-byte mask
// vector per thread); the value of a voxel is read only where the mask is non-zero, and each ROI voxel (non-NaN) feeds
// its label's row and the union row 256.
//   A  sums     the level histogram; exact rows (integer values within 2^20 of the row's minimum `base`): the 128-bit
//               sums of d^k, d = x - base, k = 1..4, the count and the sum of d over the band [band_lo, band_hi]; float
//               rows: the float64 sums of e^k, e = x - centre, and the band's count and sum of e
//   B  splits   exact rows: the count and the sum of d of the voxels with d <= split, and of the band's voxels with
//               d <= split_band; float rows: sum |x - centre| and the band's sum |x - centre_band|
// A thread accumulates the union row and the current run of its label's row in registers.  At the end of a chunk the
// lanes of a warp that hold the same row (__match_any_sync) add their values together and one lane updates the row's
// counters: in shared memory for the first kSmemSlots slots (slot 0 is the union row), with global atomics above.
// Integer counters are exact and order-independent (128-bit carry-add); float ones are order-dependent in the last bits.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/lungmask_b200.h"
#include "first_order.cuh"
#include "mask_chunk.cuh"

namespace lm {
namespace {

constexpr int kThreads = 256;
constexpr int kSmemSlots = 16;     // slots whose counters are privatised in shared memory: 16 x (88 + 1024) B
constexpr int kSumWords = 11;      // pass A counters of a slot: S1..S4 (word pairs), n_B, S_B (word pair)
constexpr unsigned kFull = 0xffffffffu;

typedef unsigned long long u64;
typedef unsigned __int128 u128;

template <typename T> constexpr bool kInt = std::is_integral<T>::value;

// The parameters of one slot (a row with a mode), in device memory.
struct FoRow {
  long long low, base, split, split_b;
  double centre, centre_b, lo, hi;
  int ng, mode, pad0, pad1;
};

// Device work area (byte offsets into FirstOrderWork::d).
struct FoDev {
  int* flag;        // bit 0: a value outside an exact row's span or a level outside 1..n_levels
  int* slot_of;     // [257]: slot of a row, -1 without a mode
  FoRow* rows;      // [slots]
  u64* hist;        // [slots][kFoLevels]
  u64* sums;        // [slots][kSumWords] (pass A) or [slots][kFoSplits] (pass B)
};

template <typename T> __device__ __forceinline__ double to_f64(T x) {
  if constexpr (std::is_same<T, __half>::value) return (double)__half2float(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return (double)__bfloat162float(x);
  else return (double)x;
}

// The fixed-bin-width level of texture.cu (lm_texture_levels_dev), restated: floor((floor(x) - low) / bw) + 1; 0 and a
// flag outside 1..ng.  x is finite here (the host refuses a row with a non-finite minimum or maximum).
template <typename T>
__device__ __forceinline__ int fo_level(T x, double xd, long long low, int bw, int ng, int* flag) {
  long long f;
  if constexpr (kInt<T>) {
    f = (long long)x;
  } else {
    const double d = floor(xd);
    if (!(d > -9.0e18 && d < 9.0e18)) { atomicOr(flag, 1); return 0; }
    f = (long long)d;
  }
  const u64 q = f < low ? 0ull : ((u64)f - (u64)low) / (unsigned)bw + 1;
  if (q < 1 || q > (u64)ng) { atomicOr(flag, 1); return 0; }
  return (int)q;
}

// 128-bit add from two 64-bit atomics (stats.cu): the carry of the low word goes into the high word.
__device__ __forceinline__ void atomic_add128(u64* p, u128 v) {
  const u64 lo = (u64)v;
  u64 hi = (u64)(v >> 64);
  if (lo) {
    const u64 old = atomicAdd(p, lo);
    if (old + lo < old) ++hi;
  }
  if (hi) atomicAdd(p + 1, hi);
}

__device__ __forceinline__ u64 shfl64(unsigned g, u64 v, int src) { return __shfl_sync(g, v, src); }
__device__ __forceinline__ u64 shfl_xor64(u64 v, int o) { return __shfl_xor_sync(kFull, v, o); }
__device__ __forceinline__ u128 shfl128(unsigned g, u128 v, int src) {
  return ((u128)shfl64(g, (u64)(v >> 64), src) << 64) | shfl64(g, (u64)v, src);
}
__device__ __forceinline__ u128 shfl_xor128(u128 v, int o) {
  return ((u128)shfl_xor64((u64)(v >> 64), o) << 64) | shfl_xor64((u64)v, o);
}
__device__ __forceinline__ double shfl_d(unsigned g, double v, int src) { return __shfl_sync(g, v, src); }
__device__ __forceinline__ double shfl_xor_d(double v, int o) { return __shfl_xor_sync(kFull, v, o); }

// The sum of v over the lanes of `group` (every lane of it calls this), valid in its lowest lane: a butterfly when the
// group is the whole warp, else the lowest lane gathers the others one by one.
template <typename V> __device__ __forceinline__ V group_sum(V v, unsigned group) {
  if (group == kFull) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      if constexpr (std::is_same<V, u128>::value) v += shfl_xor128(v, o);
      else if constexpr (std::is_same<V, double>::value) v += shfl_xor_d(v, o);
      else v += shfl_xor64(v, o);
    }
    return v;
  }
  V acc = v;
  for (unsigned rest = group & (group - 1); rest; rest &= rest - 1) {
    const int src = __ffs(rest) - 1;
    if constexpr (std::is_same<V, u128>::value) acc += shfl128(group, v, src);
    else if constexpr (std::is_same<V, double>::value) acc += shfl_d(group, v, src);
    else acc += shfl64(group, v, src);
  }
  return acc;
}

// One row's registers.  Pass A: exact rows use s1..s4 / nb / sb, float rows f1..f4 / nb / fb.  Pass B: exact rows use
// nb (n_lo), s1 (L), sb as n_lo_B and s2 as L_B; float rows f1 and fb.
struct Acc {
  u64 s1, s2, sb, nb;
  u128 s3, s4;
  double f1, f2, f3, f4, fb;
};

__device__ __forceinline__ void acc_clear(Acc& a) {
  a.s1 = a.s2 = a.sb = a.nb = 0;
  a.s3 = a.s4 = 0;
  a.f1 = a.f2 = a.f3 = a.f4 = a.fb = 0.0;
}

// The row parameters a thread keeps in registers.
struct RowP {
  long long low, base, split, split_b;
  double centre, centre_b, lo, hi;
  int ng, mode;
};

__device__ __forceinline__ RowP row_params(const FoRow* rows, int s) {
  const FoRow& r = rows[s];
  return {r.low, r.base, r.split, r.split_b, r.centre, r.centre_b, r.lo, r.hi, r.ng, r.mode};
}

template <typename T, int kPass>
__device__ __forceinline__ void acc_add(Acc& a, T x, double xd, const RowP& p, int* flag) {
  const bool band = xd >= p.lo && xd <= p.hi;
  if constexpr (kInt<T>) {
    if (p.mode == kFoExact) {
      const u64 d = (u64)(long long)x - (u64)p.base;   // modular: a value below base wraps above the span
      if (d >= (u64)kFoExactSpan) { atomicOr(flag, 1); return; }
      if constexpr (kPass == 0) {
        const u64 d2 = d * d;
        a.s1 += d;
        a.s2 += d2;
        a.s3 += (u128)(d2 * d);
        a.s4 += (u128)d2 * d2;
        if (band) { ++a.nb; a.sb += d; }
      } else {
        if ((long long)d <= p.split) { ++a.nb; a.s1 += d; }
        if (band && (long long)d <= p.split_b) { ++a.sb; a.s2 += d; }
      }
      return;
    }
  }
  if constexpr (kPass == 0) {
    const double e = xd - p.centre, e2 = e * e;
    a.f1 += e;
    a.f2 += e2;
    a.f3 += e2 * e;
    a.f4 += e2 * e2;
    if (band) { ++a.nb; a.fb += e; }
  } else {
    a.f1 += fabs(xd - p.centre);
    if (band) a.fb += fabs(xd - p.centre_b);
  }
}

// Adds a row's registers to its counters w (shared or global memory).
template <int kPass> __device__ __forceinline__ void acc_store(u64* w, const Acc& a, int mode) {
  double* wd = reinterpret_cast<double*>(w);
  if constexpr (kPass == 0) {
    if (mode == kFoExact) {
      atomic_add128(w, a.s1);
      atomic_add128(w + 2, a.s2);
      atomic_add128(w + 4, a.s3);
      atomic_add128(w + 6, a.s4);
      atomic_add128(w + 9, a.sb);
    } else {
      atomicAdd(wd, a.f1);
      atomicAdd(wd + 2, a.f2);
      atomicAdd(wd + 4, a.f3);
      atomicAdd(wd + 6, a.f4);
      atomicAdd(wd + 9, a.fb);
    }
    if (a.nb) atomicAdd(w + 8, a.nb);
  } else {
    if (mode == kFoExact) {
      if (a.nb) { atomicAdd(w, a.nb); atomicAdd(w + 1, a.s1); }
      if (a.sb) { atomicAdd(w + 2, a.sb); atomicAdd(w + 3, a.s2); }
    } else {
      atomicAdd(wd, a.f1);
      atomicAdd(wd + 2, a.fb);
    }
  }
}

// The lanes of `group` (one row, mode uniform over the group) add their registers; the lowest lane stores.
template <int kPass> __device__ __forceinline__ void acc_group_store(Acc& a, unsigned group, int mode, u64* w) {
  if (mode == kFoExact) {
    a.s1 = group_sum(a.s1, group);
    a.s2 = group_sum(a.s2, group);
    a.sb = group_sum(a.sb, group);
    a.nb = group_sum(a.nb, group);
    if constexpr (kPass == 0) {
      a.s3 = group_sum(a.s3, group);
      a.s4 = group_sum(a.s4, group);
    }
  } else {
    a.f1 = group_sum(a.f1, group);
    a.fb = group_sum(a.fb, group);
    if constexpr (kPass == 0) {
      a.f2 = group_sum(a.f2, group);
      a.f3 = group_sum(a.f3, group);
      a.f4 = group_sum(a.f4, group);
      a.nb = group_sum(a.nb, group);
    }
  }
  if ((int)(threadIdx.x & 31) == __ffs(group) - 1) acc_store<kPass>(w, a, mode);
}

// kPass 0: pass A (words = kSumWords, histograms), 1: pass B (words = kFoSplits).
// Dynamic shared memory: counters [sm][words] (u64) | histograms [sm][kFoLevels] (u32, pass A) | slot_of [257] (int).
template <typename T, int kPass>
__global__ void __launch_bounds__(kThreads) first_order_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                               size_t n, FoDev g, int slots, int bw) {
  constexpr int kWords = kPass == 0 ? kSumWords : kFoSplits;
  extern __shared__ u64 s_dyn[];
  const int sm = min(slots, kSmemSlots);
  u64* s_sum = s_dyn;
  unsigned* s_hist = reinterpret_cast<unsigned*>(s_sum + sm * kWords);
  int* s_slot = reinterpret_cast<int*>(s_hist + (kPass == 0 ? sm * kFoLevels : 0));
  for (int i = threadIdx.x; i < sm * kWords; i += blockDim.x) s_sum[i] = 0;
  if constexpr (kPass == 0)
    for (int i = threadIdx.x; i < sm * kFoLevels; i += blockDim.x) s_hist[i] = 0;
  for (int i = threadIdx.x; i < kFoRows; i += blockDim.x) s_slot[i] = g.slot_of[i];
  __syncthreads();

  auto counters = [&](int s) { return s < sm ? s_sum + (size_t)s * kWords : g.sums + (size_t)s * kWords; };
  const int us = s_slot[256];   // the union row: slot 0
  const RowP up = row_params(g.rows, us);
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    const unsigned am = __activemask();
    if (__all_sync(am, (lab.x | lab.y | lab.z | lab.w) == 0)) continue;
    Acc ua, la;
    acc_clear(ua);
    acc_clear(la);
    int ls = -1;   // the slot of the label run accumulated in `la`
    RowP lp = up;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (!l) continue;
      const T x = vol[base + k];
      const double xd = to_f64(x);
      if constexpr (!kInt<T>) {
        if (isnan(xd)) continue;
      }
      const int s = s_slot[l];   // -1: a label without a row of its own (it still feeds the union row)
      if (s >= 0) {
        if (s != ls) {
          if (ls >= 0) acc_store<kPass>(counters(ls), la, lp.mode);
          ls = s;
          lp = row_params(g.rows, s);
          acc_clear(la);
        }
        acc_add<T, kPass>(la, x, xd, lp, g.flag);
        if constexpr (kPass == 0) {
          const int ql = fo_level(x, xd, lp.low, bw, lp.ng, g.flag);
          if (ql) {
            if (s < sm) atomicAdd(&s_hist[s * kFoLevels + ql], 1u);
            else atomicAdd(&g.hist[(size_t)s * kFoLevels + ql], 1ull);
          }
        }
      }
      acc_add<T, kPass>(ua, x, xd, up, g.flag);
      if constexpr (kPass == 0) {
        const int qu = fo_level(x, xd, up.low, bw, up.ng, g.flag);
        if (qu) atomicAdd(&s_hist[us * kFoLevels + qu], 1u);
      }
    }
    acc_group_store<kPass>(ua, am, up.mode, counters(us));
    const unsigned peers = __match_any_sync(am, ls);
    if (ls >= 0) acc_group_store<kPass>(la, peers, lp.mode, counters(ls));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < sm * kWords; i += blockDim.x) {
    const int s = i / kWords, k = i % kWords;
    const int mode = g.rows[s].mode;
    u64* dst = g.sums + i;
    if (kPass == 0 && mode == kFoExact && k != 8) {   // a 128-bit pair, added by its low word's thread
      if (k == 0 || k == 2 || k == 4 || k == 6 || k == 9) {
        const u128 v = ((u128)s_sum[i + 1] << 64) | s_sum[i];
        if (v) atomic_add128(dst, v);
      }
    } else if (mode == kFoExact || (kPass == 0 && k == 8)) {
      if (s_sum[i]) atomicAdd(dst, s_sum[i]);
    } else if ((kPass == 0 && (k == 0 || k == 2 || k == 4 || k == 6 || k == 9)) || (kPass == 1 && (k == 0 || k == 2))) {
      atomicAdd(reinterpret_cast<double*>(dst), reinterpret_cast<const double*>(s_sum)[i]);
    }
  }
  if constexpr (kPass == 0)
    for (int i = threadIdx.x; i < sm * kFoLevels; i += blockDim.x)
      if (s_hist[i]) atomicAdd(&g.hist[i], (u64)s_hist[i]);
}

// ---- host ----------------------------------------------------------------------------------------------------------
#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Carves the work area for `slots` slots; returns its size (d == nullptr: size only).
size_t layout(char* d, int slots, FoDev* g) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = d ? d + off : nullptr; off += align256(bytes); return p; };
  g->flag = (int*)take(4);
  g->slot_of = (int*)take(kFoRows * 4);
  g->rows = (FoRow*)take((size_t)slots * sizeof(FoRow));
  g->hist = (u64*)take((size_t)slots * kFoLevels * 8);
  g->sums = (u64*)take((size_t)slots * kSumWords * 8);
  return off;
}

template <typename K>
int grid_for(K kernel, size_t smem, size_t n, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (n + (size_t)kThreads * kChunk - 1) / ((size_t)kThreads * kChunk);
  const size_t gr = std::min((size_t)per_sm * num_sms, need);
  return (int)std::max<size_t>(gr, 1);
}

// Slot order: the union row first (always privatised), then the labels ascending.  -> the number of slots.
int slot_table(const FirstOrderRows& r, int* slot_of, std::vector<int>& row_of) {
  row_of.clear();
  for (int i = 0; i < kFoRows; ++i) slot_of[i] = -1;
  if (r.mode[256] != kFoSkip) { slot_of[256] = 0; row_of.push_back(256); }
  for (int l = 1; l < 256; ++l)
    if (r.mode[l] != kFoSkip) { slot_of[l] = (int)row_of.size(); row_of.push_back(l); }
  return (int)row_of.size();
}

template <typename T, int kPass>
int run_pass(FirstOrderWork& w, const T* vol, const uint8_t* mask, size_t n, int bw, const FirstOrderRows& r,
             std::vector<u64>& hist, std::vector<u64>& sums, std::vector<int>& row_of, int num_sms, cudaStream_t st,
             int64_t* launches) {
  constexpr int kWords = kPass == 0 ? kSumWords : kFoSplits;
  int slot_of[kFoRows];
  const int slots = slot_table(r, slot_of, row_of);
  if (slots == 0 || slot_of[256] != 0) return slots == 0 ? 0 : -1;   // a label row needs the union row
  FoDev g;
  SC((cudaError_t)w.reserve(layout(nullptr, slots, &g)));
  layout(static_cast<char*>(w.d), slots, &g);
  std::vector<FoRow> rows(slots);
  for (int s = 0; s < slots; ++s) {
    const int i = row_of[s];
    FoRow& p = rows[s];
    p.mode = r.mode[i];
    p.low = kPass == 0 ? (long long)r.low[i] : 0;
    p.ng = kPass == 0 ? r.n_levels[i] : 0;
    p.base = (long long)r.base[i];
    p.split = kPass == 1 ? (long long)r.split[i] : 0;
    p.split_b = kPass == 1 ? (long long)r.split_band[i] : 0;
    p.centre = r.centre[i];
    p.centre_b = kPass == 1 ? r.centre_band[i] : 0.0;
    p.lo = r.band_lo[i];
    p.hi = r.band_hi[i];
    p.pad0 = p.pad1 = 0;
  }
  SC(cudaMemsetAsync(g.flag, 0, 4, st));
  SC(cudaMemcpyAsync(g.slot_of, slot_of, sizeof(slot_of), cudaMemcpyHostToDevice, st));
  SC(cudaMemcpyAsync(g.rows, rows.data(), slots * sizeof(FoRow), cudaMemcpyHostToDevice, st));
  if (kPass == 0) SC(cudaMemsetAsync(g.hist, 0, (size_t)slots * kFoLevels * 8, st));
  SC(cudaMemsetAsync(g.sums, 0, (size_t)slots * kWords * 8, st));
  const int sm = std::min(slots, kSmemSlots);
  const size_t smem = (size_t)sm * kWords * 8 + (kPass == 0 ? (size_t)sm * kFoLevels * 4 : 0) + kFoRows * 4;
  first_order_kernel<T, kPass><<<grid_for(first_order_kernel<T, kPass>, smem, n, num_sms), kThreads, smem, st>>>(
      vol, mask, n, g, slots, bw);
  SC(cudaGetLastError());
  ++*launches;
  int flag = 0;
  if (kPass == 0) {
    hist.assign((size_t)slots * kFoLevels, 0);
    SC(cudaMemcpyAsync(hist.data(), g.hist, hist.size() * 8, cudaMemcpyDeviceToHost, st));
  }
  sums.assign((size_t)slots * kWords, 0);
  SC(cudaMemcpyAsync(sums.data(), g.sums, sums.size() * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(&flag, g.flag, 4, cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? kFoRange : 0;
}

template <typename T>
int sums_t(FirstOrderWork& w, const T* vol, const uint8_t* mask, size_t n, int bw, const FirstOrderRows& r, int64_t* hist,
           uint64_t* int_sums, int64_t* band_count, double* float_sums, int num_sms, cudaStream_t st, int64_t* launches) {
  for (size_t i = 0; i < (size_t)kFoRows * kFoLevels; ++i) hist[i] = 0;
  for (size_t i = 0; i < (size_t)kFoRows * kFoIntSums; ++i) int_sums[i] = 0;
  for (size_t i = 0; i < (size_t)kFoRows * kFoFloatSums; ++i) float_sums[i] = 0.0;
  for (int i = 0; i < kFoRows; ++i) band_count[i] = 0;
  std::vector<u64> h, s;
  std::vector<int> row_of;
  const int rc = run_pass<T, 0>(w, vol, mask, n, bw, r, h, s, row_of, num_sms, st, launches);
  if (rc) return rc;
  for (size_t k = 0; k < row_of.size(); ++k) {
    const int i = row_of[k];
    const u64* c = &s[k * kSumWords];
    for (int b = 0; b < kFoLevels; ++b) hist[(size_t)i * kFoLevels + b] = (int64_t)h[k * kFoLevels + b];
    band_count[i] = (int64_t)c[8];
    if (r.mode[i] == kFoExact) {
      const int from[kFoIntSums] = {0, 1, 2, 3, 4, 5, 6, 7, 9, 10};
      for (int j = 0; j < kFoIntSums; ++j) int_sums[(size_t)i * kFoIntSums + j] = c[from[j]];
    } else {
      const double* cd = reinterpret_cast<const double*>(c);
      const int from[kFoFloatSums] = {0, 2, 4, 6, 9};
      for (int j = 0; j < kFoFloatSums; ++j) float_sums[(size_t)i * kFoFloatSums + j] = cd[from[j]];
    }
  }
  return 0;
}

template <typename T>
int splits_t(FirstOrderWork& w, const T* vol, const uint8_t* mask, size_t n, const FirstOrderRows& r, int64_t* below,
             double* abs_dev, int num_sms, cudaStream_t st, int64_t* launches) {
  for (size_t i = 0; i < (size_t)kFoRows * kFoSplits; ++i) below[i] = 0;
  for (size_t i = 0; i < (size_t)kFoRows * 2; ++i) abs_dev[i] = 0.0;
  std::vector<u64> h, s;
  std::vector<int> row_of;
  const int rc = run_pass<T, 1>(w, vol, mask, n, 1, r, h, s, row_of, num_sms, st, launches);
  if (rc) return rc;
  for (size_t k = 0; k < row_of.size(); ++k) {
    const int i = row_of[k];
    const u64* c = &s[k * kFoSplits];
    if (r.mode[i] == kFoExact) {
      for (int j = 0; j < kFoSplits; ++j) below[(size_t)i * kFoSplits + j] = (int64_t)c[j];
    } else {
      const double* cd = reinterpret_cast<const double*>(c);
      abs_dev[(size_t)i * 2] = cd[0];
      abs_dev[(size_t)i * 2 + 1] = cd[2];
    }
  }
  return 0;
}

}  // namespace

int FirstOrderWork::reserve(size_t bytes) {
  if (bytes <= d_bytes) return 0;
  release();
  const cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) { d = nullptr; return (int)e; }
  d_bytes = bytes;
  return 0;
}

void FirstOrderWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  d_bytes = 0;
}

#define LM_FO_SWITCH(CASE)                \
  switch (dtype) {                        \
    CASE(LM_DTYPE_U8, uint8_t);           \
    CASE(LM_DTYPE_I8, int8_t);            \
    CASE(LM_DTYPE_I16, int16_t);          \
    CASE(LM_DTYPE_I32, int32_t);          \
    CASE(LM_DTYPE_I64, int64_t);          \
    CASE(LM_DTYPE_F16, __half);           \
    CASE(LM_DTYPE_BF16, __nv_bfloat16);   \
    CASE(LM_DTYPE_F32, float);            \
    CASE(LM_DTYPE_F64, double);           \
    default: return -1;                   \
  }

int first_order_sums(FirstOrderWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, int bin_width,
                     const FirstOrderRows& rows, int64_t* hist, uint64_t* int_sums, int64_t* band_count, double* float_sums,
                     int num_sms, cudaStream_t st, int64_t* launches) {
#define LM_FO_SUMS(code, T)                                                                                              \
  case code:                                                                                                             \
    return sums_t<T>(w, static_cast<const T*>(d_vol), d_mask, n, bin_width, rows, hist, int_sums, band_count, float_sums, \
                     num_sms, st, launches)
  LM_FO_SWITCH(LM_FO_SUMS)
#undef LM_FO_SUMS
}

int first_order_splits(FirstOrderWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n,
                       const FirstOrderRows& rows, int64_t* below, double* abs_dev, int num_sms, cudaStream_t st,
                       int64_t* launches) {
#define LM_FO_SPLITS(code, T) \
  case code: return splits_t<T>(w, static_cast<const T*>(d_vol), d_mask, n, rows, below, abs_dev, num_sms, st, launches)
  LM_FO_SWITCH(LM_FO_SPLITS)
#undef LM_FO_SPLITS
}

}  // namespace lm
