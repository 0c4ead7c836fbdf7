// Per-label volume and HU statistics (lm_label_stats / lm_label_stats_dev, DESIGN §4.6).
//
// Passes over the (volume, mask) pair, each grid-stride over 16-voxel chunks (one 16-byte mask vector per thread); the
// value of a voxel is read only where the mask is non-zero:
//   1. count      per-label voxel and NaN counts (shared-memory privatised; integer volumes read the mask alone)
//   2. histogram  per present label: 4098 bins of floor(value) (under, -1024..3071, over), min / max as ordered keys and,
//                 for integer volumes, the exact 128-bit sums of x and x^2; shared-memory histograms up to kSmemSlots
//                 labels, global atomics above
//   3. moments    float volumes only: sums of (x - c) and (x - c)^2 in float64, c = the label's median bin
//   4. select     radix select of the order statistics that the histogram does not pin down exactly (any bin of a float
//                 volume, the under / overflow bins of an integer one): 8-bit digits of the ordered key, restricted to
//                 the row and the bin, a few passes over the volume with one digit scan per pass
// The host synchronises after passes 1 and 2 (it sizes the next pass from the counts) and at the end.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/lungmask_b200.h"
#include "mask_chunk.cuh"
#include "stats.cuh"

namespace lm {
namespace {

constexpr int kThreads = 512;
constexpr int kSmemSlots = 12;      // labels whose histograms are privatised in shared memory: 12 x 4098 x 4 B = 192 KB
constexpr int kSmemTargets = 96;    // selection targets whose digit histograms fit shared memory: 96 x 256 x 4 B = 96 KB
constexpr int kMaxSlots = 255;      // labels 1..255
constexpr unsigned long long kSign = 0x8000000000000000ull;
constexpr unsigned kFull = 0xffffffffu;

typedef unsigned long long u64;
typedef unsigned __int128 u128;

template <typename T> constexpr bool kInt = std::is_integral<T>::value;
template <typename T> constexpr bool kF64 = std::is_same<T, double>::value;

// One order statistic to refine: the element of rank `rank` (0-based, among the non-NaN values of `row` in bin `bin`).
// The ordered key is known above bit shift + 8 (prefix); the pass finds the digit at [shift, shift + 8).  shift < 0: done,
// the key is `prefix`.
struct SelTarget {
  u64 prefix;
  u64 rank;
  int row, bin, shift, pad;
};

// Device work area (byte offsets into LabelStatsWork::d).
struct StatsDev {
  u64 *cnt, *nan;          // [256]
  int* slot_of;            // [256]: slot of a present label
  u64* hist;               // [slots][kStatsBins]
  u64 *kmin, *kmax;        // [slots] ordered keys
  u64* sums;               // [slots][4]: 128-bit sum of x, 128-bit sum of x^2 (integer volumes)
  double* mom;             // [slots][2]: sum of (x - c), sum of (x - c)^2 (float volumes)
  double* shift;           // [slots]: c
  SelTarget* tg;           // [targets]
  int* tfirst;             // [258]: targets of row r are tg[tfirst[r] .. tfirst[r + 1])
  u64* thist;              // [targets][256]
};

// ---- values: ordered keys (unsigned order = value order), bins, NaN ------------------------------------------------
__host__ __device__ inline u64 key_i64(long long v) { return (u64)v ^ kSign; }
__host__ __device__ inline u64 key_f32(float f) {
  unsigned u;
  memcpy(&u, &f, 4);
  return (u >> 31) ? (u64)(~u) : (u64)(u | 0x80000000u);
}
__host__ __device__ inline u64 key_f64(double d) {
  u64 b;
  memcpy(&b, &d, 8);
  return (b >> 63) ? ~b : (b | kSign);
}

template <typename T> __device__ __forceinline__ float to_f32(T x) {
  if constexpr (std::is_same<T, __half>::value) return __half2float(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat162float(x);
  else return (float)x;
}
template <typename T> __device__ __forceinline__ double to_f64(T x) {
  if constexpr (kF64<T>) return x;
  else if constexpr (kInt<T>) return (double)x;
  else return (double)to_f32(x);
}
// float16 / bfloat16 / float32 values use the 32-bit float key (exact: they are floats), float64 the 64-bit one.
template <typename T> __device__ __forceinline__ u64 key_of(T x) {
  if constexpr (kInt<T>) return key_i64((long long)x);
  else if constexpr (kF64<T>) return key_f64(x);
  else return key_f32(to_f32(x));
}
template <typename T> __device__ __forceinline__ bool is_nan(T x) {
  if constexpr (kInt<T>) return false;
  else return isnan(to_f64(x));
}
// floor(value) -> bin; for integer t, floor(x) < t <=> x < t, so the cumulative histogram gives count(x < t) exactly.
template <typename T> __device__ __forceinline__ int bin_of(T x) {
  if constexpr (kInt<T>) {
    const long long v = (long long)x;
    return v < -1024 ? 0 : (v > 3071 ? kStatsBins - 1 : (int)v + 1025);
  } else {
    const double d = to_f64(x);
    return d < -1024.0 ? 0 : (d >= 3072.0 ? kStatsBins - 1 : (int)floor(d) + 1025);
  }
}

// 128-bit modular add from two 64-bit atomics: the carry of the low word goes into the high word, so the sum is exact
// and independent of the order of the adds.
__device__ __forceinline__ void atomic_add128(u64* p, u128 v) {
  const u64 lo = (u64)v;
  u64 hi = (u64)(v >> 64);
  if (lo) {
    const u64 old = atomicAdd(p, lo);
    if (old + lo < old) ++hi;
  }
  if (hi) atomicAdd(p + 1, hi);
}

__device__ __forceinline__ u64 shfl_xor64(u64 v, int o) { return __shfl_xor_sync(kFull, v, o); }
__device__ __forceinline__ u128 shfl_xor128(u128 v, int o) {
  return ((u128)shfl_xor64((u64)(v >> 64), o) << 64) | shfl_xor64((u64)v, o);
}

// ---- 1. counts ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) stats_count_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                               size_t n, u64* __restrict__ cnt, u64* __restrict__ nan) {
  __shared__ unsigned s_cnt[256], s_nan[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cnt[i] = s_nan[i] = 0;
  __syncthreads();
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    int run = 0;
    unsigned rn = 0, rnan = 0;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (l != run) {
        if (run) { atomicAdd(&s_cnt[run], rn); if (rnan) atomicAdd(&s_nan[run], rnan); }
        run = l;
        rn = rnan = 0;
      }
      if (l) {
        ++rn;
        if constexpr (!kInt<T>) rnan += is_nan(vol[base + k]) ? 1u : 0u;
      }
    }
    // the warp's lanes mostly end on the same label: one shared atomic per label and warp
    const unsigned am = __activemask();
    const unsigned peers = __match_any_sync(am, run);
    const unsigned tn = __reduce_add_sync(peers, rn), tnan = __reduce_add_sync(peers, rnan);
    if (run && (int)(threadIdx.x & 31) == __ffs(peers) - 1) {
      atomicAdd(&s_cnt[run], tn);
      if (tnan) atomicAdd(&s_nan[run], tnan);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x + 1; i < 256; i += blockDim.x) {
    if (s_cnt[i]) atomicAdd(&cnt[i], (u64)s_cnt[i]);
    if (s_nan[i]) atomicAdd(&nan[i], (u64)s_nan[i]);
  }
}

// ---- 2. histograms, min / max, exact integer sums -----------------------------------------------------------------
// Dynamic shared memory: kmin | kmax | sums [slots][4] (u64) | slot_of [256] (int) | hist [slots][kStatsBins] (u32, kSmem).
template <typename T, bool kSmem>
__global__ void __launch_bounds__(kThreads) stats_hist_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                              size_t n, StatsDev g, int slots) {
  extern __shared__ u64 s_dyn[];
  u64* s_min = s_dyn;
  u64* s_max = s_min + slots;
  u64* s_sum = s_max + slots;
  int* s_slot = reinterpret_cast<int*>(s_sum + 4 * slots);
  unsigned* s_hist = reinterpret_cast<unsigned*>(s_slot + 256);
  for (int i = threadIdx.x; i < slots; i += blockDim.x) { s_min[i] = ~0ull; s_max[i] = 0; }
  for (int i = threadIdx.x; i < 4 * slots; i += blockDim.x) s_sum[i] = 0;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_slot[i] = g.slot_of[i];
  if constexpr (kSmem)
    for (int i = threadIdx.x; i < slots * kStatsBins; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();

  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    int rs = -1;   // the slot of the run of equal labels this thread accumulates in registers
    u64 rmin = ~0ull, rmax = 0;
    u128 r1 = 0, r2 = 0;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      if (label_at(lab, k)) {
        const T x = vol[base + k];
        if (!is_nan(x)) {
          const int s = s_slot[label_at(lab, k)];
          if (s != rs) {
            if (rs >= 0) {
              atomicMin(&s_min[rs], rmin);
              atomicMax(&s_max[rs], rmax);
              if constexpr (kInt<T>) { atomic_add128(&s_sum[4 * rs], r1); atomic_add128(&s_sum[4 * rs + 2], r2); }
            }
            rs = s;
            rmin = ~0ull;
            rmax = 0;
            r1 = r2 = 0;
          }
          const u64 key = key_of(x);
          rmin = key < rmin ? key : rmin;
          rmax = key > rmax ? key : rmax;
          if constexpr (kInt<T>) {
            const long long v = (long long)x;
            r1 += (u128)(__int128)v;
            r2 += (u128)((__int128)v * v);
          }
          const int b = bin_of(x);
          if constexpr (kSmem) atomicAdd(&s_hist[s * kStatsBins + b], 1u);
          else atomicAdd(&g.hist[(size_t)s * kStatsBins + b], 1ull);
        }
      }
    }
    // warp-uniform run (the common case inside an organ): reduce in registers, one lane updates shared memory
    const unsigned am = __activemask();
    const int r0 = __shfl_sync(am, rs, __ffs(am) - 1);
    if (am == kFull && __all_sync(kFull, rs == r0)) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const u64 a = shfl_xor64(rmin, o), b = shfl_xor64(rmax, o);
        rmin = a < rmin ? a : rmin;
        rmax = b > rmax ? b : rmax;
        if constexpr (kInt<T>) { r1 += shfl_xor128(r1, o); r2 += shfl_xor128(r2, o); }
      }
      if ((threadIdx.x & 31) != 0) rs = -1;
    }
    if (rs >= 0) {
      atomicMin(&s_min[rs], rmin);
      atomicMax(&s_max[rs], rmax);
      if constexpr (kInt<T>) { atomic_add128(&s_sum[4 * rs], r1); atomic_add128(&s_sum[4 * rs + 2], r2); }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < slots; i += blockDim.x) {
    if (s_min[i] != ~0ull) atomicMin(&g.kmin[i], s_min[i]);
    if (s_max[i] != 0) atomicMax(&g.kmax[i], s_max[i]);
  }
  if constexpr (kInt<T>)
    for (int i = threadIdx.x; i < 2 * slots; i += blockDim.x) {
      const u128 v = ((u128)s_sum[2 * i + 1] << 64) | s_sum[2 * i];
      if (v) atomic_add128(&g.sums[2 * i], v);
    }
  if constexpr (kSmem)
    for (int i = threadIdx.x; i < slots * kStatsBins; i += blockDim.x)
      if (s_hist[i]) atomicAdd(&g.hist[i], (u64)s_hist[i]);
}

// ---- 3. shifted moments of float volumes ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) stats_moments_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                                 size_t n, StatsDev g) {
  __shared__ int s_slot[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_slot[i] = g.slot_of[i];
  __syncthreads();
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    int rs = -1;
    double c0 = 0.0, r1 = 0.0, r2 = 0.0;
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      if (label_at(lab, k)) {
        const T x = vol[base + k];
        if (!is_nan(x)) {
          const int s = s_slot[label_at(lab, k)];
          if (s != rs) {
            if (rs >= 0) { atomicAdd(&g.mom[2 * rs], r1); atomicAdd(&g.mom[2 * rs + 1], r2); }
            rs = s;
            c0 = g.shift[s];
            r1 = r2 = 0.0;
          }
          const double d = to_f64(x) - c0;
          r1 += d;
          r2 += d * d;
        }
      }
    }
    const unsigned am = __activemask();
    const int r0 = __shfl_sync(am, rs, __ffs(am) - 1);
    if (am == kFull && __all_sync(kFull, rs == r0)) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        r1 += __shfl_xor_sync(kFull, r1, o);
        r2 += __shfl_xor_sync(kFull, r2, o);
      }
      if ((threadIdx.x & 31) != 0) rs = -1;
    }
    if (rs >= 0) { atomicAdd(&g.mom[2 * rs], r1); atomicAdd(&g.mom[2 * rs + 1], r2); }
  }
}

// ---- 4. radix select ------------------------------------------------------------------------------------------------
// kSmem: dynamic shared memory holds targets [ntg] | tfirst [258] | digit histograms [ntg][256] (u32).  Otherwise it holds
// tfirst alone and the targets and histograms stay in global memory (any number of targets).
template <typename T, bool kSmem>
__global__ void __launch_bounds__(kThreads) stats_select_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                                size_t n, StatsDev g, int ntg) {
  extern __shared__ u64 s_dyn[];
  SelTarget* s_tg = reinterpret_cast<SelTarget*>(s_dyn);
  int* s_first = reinterpret_cast<int*>(kSmem ? s_tg + ntg : s_tg);
  unsigned* s_h = reinterpret_cast<unsigned*>(s_first + 258);
  const SelTarget* tgs = kSmem ? s_tg : g.tg;
  if constexpr (kSmem) {
    for (int i = threadIdx.x; i < ntg; i += blockDim.x) s_tg[i] = g.tg[i];
    for (int i = threadIdx.x; i < ntg * 256; i += blockDim.x) s_h[i] = 0;
  }
  for (int i = threadIdx.x; i < 258; i += blockDim.x) s_first[i] = g.tfirst[i];
  __syncthreads();
  const int u0 = s_first[256], u1 = s_first[257];
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (!l) continue;
      const int t0 = s_first[l], t1 = s_first[l + 1];
      if (t0 == t1 && u0 == u1) continue;
      const T x = vol[base + k];
      if (is_nan(x)) continue;
      const u64 key = key_of(x);
      const int b = bin_of(x);
      for (int pass = 0; pass < 2; ++pass) {
        const int e0 = pass ? u0 : t0, e1 = pass ? u1 : t1;
        for (int t = e0; t < e1; ++t) {
          const SelTarget& tg = tgs[t];
          if (tg.shift < 0 || tg.bin != b || (((key ^ tg.prefix) >> tg.shift) >> 8) != 0) continue;
          const int d = (int)((key >> tg.shift) & 255);
          if constexpr (kSmem) atomicAdd(&s_h[t * 256 + d], 1u);
          else atomicAdd(&g.thist[(size_t)t * 256 + d], 1ull);
        }
      }
    }
  }
  if constexpr (kSmem) {
    __syncthreads();
    for (int i = threadIdx.x; i < ntg * 256; i += blockDim.x)
      if (s_h[i]) atomicAdd(&g.thist[i], (u64)s_h[i]);
  }
}

// One thread per target: the digit that holds the target's rank, then the next (lower) digit; clears the histogram.
__global__ void stats_select_scan_kernel(StatsDev g, int ntg) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntg) return;
  SelTarget tg = g.tg[t];
  if (tg.shift < 0) return;
  u64* h = g.thist + (size_t)t * 256;
  u64 below = 0;
  int d = 0;
  for (; d < 255; ++d) {
    const u64 c = h[d];
    if (below + c > tg.rank) break;
    below += c;
  }
  for (int i = 0; i < 256; ++i) h[i] = 0;
  tg.rank -= below;
  tg.prefix |= (u64)d << tg.shift;
  tg.shift -= 8;
  g.tg[t] = tg;
}

// ---- host ----------------------------------------------------------------------------------------------------------
#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Carves the work area; returns its size (d == nullptr: size only).
size_t layout(char* d, int max_targets, StatsDev* g) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = d ? d + off : nullptr; off += align256(bytes); return p; };
  g->cnt = (u64*)take(256 * 8);
  g->nan = (u64*)take(256 * 8);
  g->slot_of = (int*)take(256 * 4);
  g->hist = (u64*)take((size_t)kMaxSlots * kStatsBins * 8);
  g->kmin = (u64*)take(kMaxSlots * 8);
  g->kmax = (u64*)take(kMaxSlots * 8);
  g->sums = (u64*)take(kMaxSlots * 4 * 8);
  g->mom = (double*)take(kMaxSlots * 2 * 8);
  g->shift = (double*)take(kMaxSlots * 8);
  g->tfirst = (int*)take(258 * 4);
  g->tg = (SelTarget*)take((size_t)max_targets * sizeof(SelTarget));
  g->thist = (u64*)take((size_t)max_targets * 256 * 8);
  return off;
}

template <typename K>
int grid_for(K kernel, size_t smem, size_t n, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (n + (size_t)kThreads * kChunk - 1) / ((size_t)kThreads * kChunk);
  const size_t g = std::min((size_t)per_sm * num_sms, need);
  return (int)std::max<size_t>(g, 1);
}

// 0: integer keys, 1: 32-bit float keys, 2: 64-bit float keys
template <typename T> constexpr int kKeyKind = kInt<T> ? 0 : (kF64<T> ? 2 : 1);

u64 host_key(int kind, double v) {
  if (kind == 0) return key_i64((long long)v);
  if (kind == 1) return key_f32((float)v);
  return key_f64(v);
}
double decode_key(int kind, u64 k) {
  if (kind == 0) return (double)(long long)(k ^ kSign);
  if (kind == 1) {
    unsigned u = (unsigned)k;
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    memcpy(&f, &u, 4);
    return (double)f;
  }
  const u64 b = (k & kSign) ? (k & ~kSign) : ~k;
  double d;
  memcpy(&d, &b, 8);
  return d;
}
// The largest value below `v` in the key's float format (the top of a bin [v - 1, v)).
double below(int kind, double v) { return kind == 1 ? (double)nextafterf((float)v, -INFINITY) : nextafter(v, -INFINITY); }

// numpy's _lerp (numpy/lib/_function_base_impl.py), each product rounded on its own: no FMA contraction.
double np_lerp(double a, double b, double t) {
  const double diff = b - a;
  volatile double p = diff * t;
  double r = a + p;
  if (t >= 0.5) {
    volatile double p2 = diff * (1.0 - t);
    r = b - p2;
  }
  return r;
}

template <typename T>
int label_stats_t(LabelStatsWork& w, const T* vol, const uint8_t* mask, size_t n, const double* q, int n_q, const int* th,
                  int n_t, const LabelStatsOut& out, int num_sms, cudaStream_t st, int64_t* launches) {
  const int kind = kKeyKind<T>;
  const int max_targets = kStatsRows * 2 * (n_q > 0 ? n_q : 1);
  StatsDev g;
  SC((cudaError_t)w.reserve(layout(nullptr, max_targets, &g)));
  layout(static_cast<char*>(w.d), max_targets, &g);
  const double qnan = NAN;
  for (int r = 0; r < kStatsRows; ++r) {
    out.voxels[r] = 0;
    out.nan_voxels[r] = 0;
    for (int k = 0; k < 4; ++k) out.moments[r * 4 + k] = qnan;
    for (int k = 0; k < n_q; ++k) out.percentile[(size_t)r * n_q + k] = qnan;
    for (int k = 0; k < n_t; ++k) out.below[(size_t)r * n_t + k] = 0;
  }

  // 1. counts
  SC(cudaMemsetAsync(g.cnt, 0, 256 * 8, st));
  SC(cudaMemsetAsync(g.nan, 0, 256 * 8, st));
  stats_count_kernel<T><<<grid_for(stats_count_kernel<T>, 0, n, num_sms), kThreads, 0, st>>>(vol, mask, n, g.cnt, g.nan);
  SC(cudaGetLastError());
  ++*launches;
  u64 cnt[256], nanc[256];
  SC(cudaMemcpyAsync(cnt, g.cnt, sizeof(cnt), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(nanc, g.nan, sizeof(nanc), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  int slot_of[256], label_of[kMaxSlots];
  int slots = 0;
  u64 fg = 0, fg_nan = 0;
  for (int l = 0; l < 256; ++l) {
    slot_of[l] = -1;
    if (l == 0 || cnt[l] == 0) continue;
    slot_of[l] = slots;
    label_of[slots++] = l;
    out.voxels[l] = (int64_t)cnt[l];
    out.nan_voxels[l] = (int64_t)nanc[l];
    fg += cnt[l];
    fg_nan += nanc[l];
  }
  out.voxels[0] = (int64_t)(n - fg);
  out.voxels[256] = (int64_t)fg;
  out.nan_voxels[256] = (int64_t)fg_nan;
  if (slots == 0) return 0;

  // 2. histograms
  SC(cudaMemcpyAsync(g.slot_of, slot_of, sizeof(slot_of), cudaMemcpyHostToDevice, st));
  SC(cudaMemsetAsync(g.hist, 0, (size_t)slots * kStatsBins * 8, st));
  SC(cudaMemsetAsync(g.kmin, 0xff, slots * 8, st));
  SC(cudaMemsetAsync(g.kmax, 0, slots * 8, st));
  SC(cudaMemsetAsync(g.sums, 0, slots * 4 * 8, st));
  const size_t smem_base = (size_t)slots * 6 * 8 + 256 * 4;
  if (slots <= kSmemSlots) {
    const size_t smem = smem_base + (size_t)slots * kStatsBins * 4;
    SC(cudaFuncSetAttribute(stats_hist_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stats_hist_kernel<T, true><<<grid_for(stats_hist_kernel<T, true>, smem, n, num_sms), kThreads, smem, st>>>(vol, mask, n, g, slots);
  } else {
    stats_hist_kernel<T, false><<<grid_for(stats_hist_kernel<T, false>, smem_base, n, num_sms), kThreads, smem_base, st>>>(
        vol, mask, n, g, slots);
  }
  SC(cudaGetLastError());
  ++*launches;
  std::vector<u64> hist((size_t)slots * kStatsBins), kmin(slots), kmax(slots), sums((size_t)slots * 4);
  SC(cudaMemcpyAsync(hist.data(), g.hist, hist.size() * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(kmin.data(), g.kmin, slots * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(kmax.data(), g.kmax, slots * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(sums.data(), g.sums, sums.size() * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));

  // rows: the present labels, then the union (its histogram is the sum of theirs)
  struct Row { int r; const u64* h; int64_t nv; u64 kmin, kmax; };
  std::vector<u64> uhist(kStatsBins, 0);
  std::vector<Row> rows;
  u64 ukmin = ~0ull, ukmax = 0;
  for (int s = 0; s < slots; ++s) {
    const int l = label_of[s];
    rows.push_back({l, &hist[(size_t)s * kStatsBins], (int64_t)(cnt[l] - nanc[l]), kmin[s], kmax[s]});
    for (int b = 0; b < kStatsBins; ++b) uhist[b] += hist[(size_t)s * kStatsBins + b];
    if (cnt[l] > nanc[l]) { ukmin = std::min(ukmin, kmin[s]); ukmax = std::max(ukmax, kmax[s]); }
  }
  rows.push_back({256, uhist.data(), (int64_t)(fg - fg_nan), ukmin, ukmax});

  // order statistics: an interior bin of an integer volume is the value; everything else becomes a selection target
  struct Pick { bool exact; double v; int target; };
  std::vector<Pick> picks((size_t)kStatsRows * n_q * 2);
  std::map<std::pair<int, u64>, int> target_of;   // (row, rank) -> target
  std::vector<SelTarget> tgs;
  std::vector<double> median_bin(slots, 0.0);
  for (const Row& row : rows) {
    if (row.nv == 0) continue;
    std::vector<u64> cum(kStatsBins + 1, 0);   // cum[b] = count of bins < b
    for (int b = 0; b < kStatsBins; ++b) cum[b + 1] = cum[b] + row.h[b];
    for (int k = 0; k < n_t; ++k) out.below[(size_t)row.r * n_t + k] = (int64_t)cum[th[k] + 1025];
    out.moments[row.r * 4 + 2] = decode_key(kind, row.kmin);
    out.moments[row.r * 4 + 3] = decode_key(kind, row.kmax);
    auto bin_of_rank = [&](u64 rank) { return (int)(std::upper_bound(cum.begin(), cum.end(), rank) - cum.begin()) - 1; };
    if (row.r < 256) {
      const int b = bin_of_rank((u64)(row.nv - 1) / 2);
      median_bin[slot_of[row.r]] = b == 0 ? -1025.0 : (double)(b - 1025);
    }
    for (int k = 0; k < n_q; ++k) {
      const double h = (double)(row.nv - 1) * (q[k] / 100.0);
      const u64 prev = h >= (double)(row.nv - 1) ? (u64)(row.nv - 1) : (u64)floor(h);
      for (int j = 0; j < 2; ++j) {
        const u64 rank = (j && h < (double)(row.nv - 1)) ? prev + 1 : prev;
        Pick& p = picks[((size_t)row.r * n_q + k) * 2 + j];
        const int b = bin_of_rank(rank);
        if (kind == 0 && b > 0 && b < kStatsBins - 1) { p = {true, (double)(b - 1025), -1}; continue; }
        auto it = target_of.find({row.r, rank});
        if (it != target_of.end()) { p = {false, 0.0, it->second}; continue; }
        // the bin's key range: its lowest and highest possible keys, narrowed to the row's min / max
        u64 lo = row.kmin, hi = row.kmax;
        if (b > 0 && b < kStatsBins - 1) {
          const double v0 = (double)(b - 1025);
          lo = std::max(lo, host_key(kind, v0 == 0.0 ? -0.0 : v0));
          hi = std::min(hi, host_key(kind, below(kind, v0 + 1.0)));
        } else if (b == 0) {
          hi = std::min(hi, kind == 0 ? key_i64(-1025) : host_key(kind, below(kind, -1024.0)));
        } else {
          lo = std::max(lo, host_key(kind, 3072.0));
        }
        const int v = (lo == hi) ? 0 : 64 - __builtin_clzll(lo ^ hi);
        const int v8 = (v + 7) / 8 * 8;
        SelTarget t;
        t.prefix = v8 >= 64 ? 0 : (lo >> v8) << v8;
        t.rank = rank - cum[b];
        t.row = row.r;
        t.bin = b;
        t.shift = v8 - 8;
        t.pad = 0;
        target_of[{row.r, rank}] = (int)tgs.size();
        p = {false, 0.0, (int)tgs.size()};
        tgs.push_back(t);
      }
    }
  }

  // 3. moments of float volumes, 4. selection
  if constexpr (!kInt<T>) {
    SC(cudaMemcpyAsync(g.shift, median_bin.data(), slots * 8, cudaMemcpyHostToDevice, st));
    SC(cudaMemsetAsync(g.mom, 0, slots * 2 * 8, st));
    stats_moments_kernel<T><<<grid_for(stats_moments_kernel<T>, 0, n, num_sms), kThreads, 0, st>>>(vol, mask, n, g);
    SC(cudaGetLastError());
    ++*launches;
  }
  const int ntg = (int)tgs.size();
  std::vector<int> perm(ntg);   // targets sorted by row: tg[tfirst[r] .. tfirst[r + 1]) belong to row r
  for (int i = 0; i < ntg; ++i) perm[i] = i;
  std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) { return tgs[a].row < tgs[b].row; });
  std::vector<int> pos(ntg);
  std::vector<SelTarget> sorted(ntg);
  int passes = 0;
  for (int i = 0; i < ntg; ++i) {
    sorted[i] = tgs[perm[i]];
    pos[perm[i]] = i;
    passes = std::max(passes, sorted[i].shift / 8 + 1);
  }
  if (ntg > 0 && passes > 0) {
    int tfirst[258];
    for (int r = 0, i = 0; r <= 257; ++r) {
      while (i < ntg && sorted[i].row < r) ++i;
      tfirst[r] = i;
    }
    SC(cudaMemcpyAsync(g.tg, sorted.data(), ntg * sizeof(SelTarget), cudaMemcpyHostToDevice, st));
    SC(cudaMemcpyAsync(g.tfirst, tfirst, sizeof(tfirst), cudaMemcpyHostToDevice, st));
    SC(cudaMemsetAsync(g.thist, 0, (size_t)ntg * 256 * 8, st));
    const bool smem_h = ntg <= kSmemTargets;
    const size_t smem = smem_h ? (size_t)ntg * (sizeof(SelTarget) + 256 * 4) + 258 * 4 : 258 * 4;
    if (smem_h) SC(cudaFuncSetAttribute(stats_select_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = smem_h ? grid_for(stats_select_kernel<T, true>, smem, n, num_sms)
                            : grid_for(stats_select_kernel<T, false>, smem, n, num_sms);
    for (int p = 0; p < passes; ++p) {
      if (smem_h) stats_select_kernel<T, true><<<grid, kThreads, smem, st>>>(vol, mask, n, g, ntg);
      else stats_select_kernel<T, false><<<grid, kThreads, smem, st>>>(vol, mask, n, g, ntg);
      stats_select_scan_kernel<<<(ntg + 127) / 128, 128, 0, st>>>(g, ntg);
      SC(cudaGetLastError());
      *launches += 2;
    }
    SC(cudaMemcpyAsync(sorted.data(), g.tg, ntg * sizeof(SelTarget), cudaMemcpyDeviceToHost, st));
  }
  std::vector<double> mom((size_t)slots * 2, 0.0);
  if (kind != 0) SC(cudaMemcpyAsync(mom.data(), g.mom, mom.size() * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));

  // mean / std.  Integer volumes: from the exact sums (the union's sums are the labels' sums).  Float volumes: per label
  // from the moments about c, the union by the pairwise combination of the labels' means and squared deviations.
  if (kind == 0) {
    u128 u1 = 0, u2 = 0;
    for (int s = 0; s <= slots; ++s) {
      const bool uni = s == slots;
      const int r = uni ? 256 : label_of[s];
      const int64_t nv = uni ? (int64_t)(fg - fg_nan) : (int64_t)cnt[r];
      const u128 s1 = uni ? u1 : (((u128)sums[4 * s + 1] << 64) | sums[4 * s]);
      const u128 s2 = uni ? u2 : (((u128)sums[4 * s + 3] << 64) | sums[4 * s + 2]);
      if (!uni) { u1 += s1; u2 += s2; }
      const __int128 si = (__int128)s1;
      const bool small = si > -((__int128)1 << 53) && si < ((__int128)1 << 53);
      out.moments[r * 4] = small ? (double)(long long)si / (double)nv : (double)((long double)si / (long double)nv);
      const long double m = (long double)si / (long double)nv;
      long double var = (long double)s2 / (long double)nv - m * m;
      out.moments[r * 4 + 1] = (double)sqrtl(var > 0 ? var : 0.0L);
    }
  } else {
    long double tot = 0.0L;
    int64_t ntot = 0;
    std::vector<double> mean(slots), m2(slots);
    for (int s = 0; s < slots; ++s) {
      const int l = label_of[s];
      const int64_t nv = (int64_t)(cnt[l] - nanc[l]);
      if (nv == 0) continue;
      mean[s] = median_bin[s] + mom[2 * s] / (double)nv;
      m2[s] = mom[2 * s + 1] - mom[2 * s] * (mom[2 * s] / (double)nv);
      out.moments[l * 4] = mean[s];
      out.moments[l * 4 + 1] = sqrt(std::max(m2[s], 0.0) / (double)nv);
      tot += (long double)median_bin[s] * nv + mom[2 * s];
      ntot += nv;
    }
    if (ntot > 0) {
      const double mu = (double)(tot / ntot);
      double m2u = 0.0;
      for (int s = 0; s < slots; ++s) {
        const int64_t nv = (int64_t)(cnt[label_of[s]] - nanc[label_of[s]]);
        if (nv) m2u += m2[s] + (double)nv * (mean[s] - mu) * (mean[s] - mu);
      }
      out.moments[256 * 4] = mu;
      out.moments[256 * 4 + 1] = sqrt(std::max(m2u, 0.0) / (double)ntot);
    }
  }

  // percentiles: numpy's indices, gamma and _lerp on the two order statistics
  for (const Row& row : rows) {
    if (row.nv == 0) continue;
    for (int k = 0; k < n_q; ++k) {
      double ab[2];
      for (int j = 0; j < 2; ++j) {
        const Pick& p = picks[((size_t)row.r * n_q + k) * 2 + j];
        ab[j] = p.exact ? p.v : decode_key(kind, sorted[pos[p.target]].prefix);
      }
      const double h = (double)(row.nv - 1) * (q[k] / 100.0);
      // numpy marks an index at or past the last element as -1 (the last one), and gamma = h - that index
      const double prev = h >= (double)(row.nv - 1) ? -1.0 : floor(h);
      out.percentile[(size_t)row.r * n_q + k] = np_lerp(ab[0], ab[1], h - prev);
    }
  }
  return 0;
}

}  // namespace

int LabelStatsWork::reserve(size_t bytes) {
  if (bytes <= d_bytes) return 0;
  release();
  const cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) { d = nullptr; return (int)e; }
  d_bytes = bytes;
  return 0;
}

void LabelStatsWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  d_bytes = 0;
}

int label_stats(LabelStatsWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, const double* q, int n_q,
                const int* t, int n_t, const LabelStatsOut& out, int num_sms, cudaStream_t st, int64_t* launches) {
#define LM_STATS_CASE(code, T) \
  case code: return label_stats_t<T>(w, static_cast<const T*>(d_vol), d_mask, n, q, n_q, t, n_t, out, num_sms, st, launches)
  switch (dtype) {
    LM_STATS_CASE(LM_DTYPE_U8, uint8_t);
    LM_STATS_CASE(LM_DTYPE_I8, int8_t);
    LM_STATS_CASE(LM_DTYPE_I16, int16_t);
    LM_STATS_CASE(LM_DTYPE_I32, int32_t);
    LM_STATS_CASE(LM_DTYPE_I64, int64_t);
    LM_STATS_CASE(LM_DTYPE_F16, __half);
    LM_STATS_CASE(LM_DTYPE_BF16, __nv_bfloat16);
    LM_STATS_CASE(LM_DTYPE_F32, float);
    LM_STATS_CASE(LM_DTYPE_F64, double);
    default: return -1;
  }
#undef LM_STATS_CASE
}

}  // namespace lm
