// Grey-level texture matrices of one ROI (lm_texture_levels_dev, lm_glcm_dev, lm_glrlm_dev, lm_neighbour_counts_dev,
// DESIGN §4.9).
//
//   levels  reads the mask as 16-byte vectors and the value only under the row; writes the row's discretised level (0
//           outside the ROI) 16 bytes at a time, the last partial chunk byte by byte.  A level outside 1..n_levels or a
//           non-finite value raises a flag instead of being written.
//   glcm    one warp per 32-voxel run along x, one lane per voxel: for each of the 13 directions d the lane reads the
//           level of v + d, and the lanes holding equal pair keys (i <= j) add their count with one atomic
//           (__match_any_sync).  Parenchyma fills a few near-diagonal bins, so the counters are privatised in shared
//           memory: the whole upper triangle of every direction while n_levels <= kSmemLevels, above that the band
//           j - i < kBand (where nearly all pairs of neighbouring voxels fall) with the rest going to global atomics.
//   glrlm   the same layout: for each direction d a lane whose voxel starts a run (its predecessor v - d is outside the
//           array, outside the ROI or at another level) walks along d to the run's end and counts the run once; lanes
//           with equal (level, length) keys add with one atomic.  Runs up to a length derived from n_levels are counted
//           in shared memory, longer ones with global atomics.
//   neighbour  the same layout: each ROI voxel reads its 26 neighbours and forms, in registers, W (neighbours in the
//           ROI), S (the sum of their levels) and c (those within alpha of its level); G(i, c), N(i, W) and
//           A(i, W) += |W i - S| are warp-aggregated by key into shared counters that hold every level.
//   glcm_offsets, neighbour_offsets  the glcm and neighbour layouts over a caller's offset list (lm_glcm_offsets_dev,
//           lm_neighbour_offsets_dev, DESIGN §4.18): distances 1..3 and in-plane neighbourhoods.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/lungmask_b200.h"
#include "mask_chunk.cuh"
#include "texture.cuh"

namespace lm {
namespace {

constexpr int kThreads = 512;
constexpr int kSmemLevels = 90;    // triangle of 13 directions: 13 x 4095 x 4 B = 212,940 B
constexpr int kBand = 16;          // n_levels > kSmemLevels: 13 x 255 x 16 x 4 B = 212,160 B
constexpr unsigned kFull = 0xffffffffu;
constexpr int kSmemWords = 53235;  // the shared budget of the GLCM triangle, 212,940 B, in 4-byte counters

// ---- levels ---------------------------------------------------------------------------------------------------------
// flag bit 0: a level outside 1..n_levels, bit 1: a non-finite value.
template <typename T>
__device__ __forceinline__ int level_of(T x, long long low, int bw, int ng, int* flag) {
  long long f;
  if constexpr (std::is_integral<T>::value) {
    f = (long long)x;
  } else {
    double d;
    if constexpr (std::is_same<T, __half>::value) d = (double)__half2float(x);
    else if constexpr (std::is_same<T, __nv_bfloat16>::value) d = (double)__bfloat162float(x);
    else d = (double)x;
    if (isnan(d)) return 0;
    if (isinf(d)) { atomicOr(flag, 2); return 0; }
    d = floor(d);
    if (d < -9.0e18 || d > 9.0e18) { atomicOr(flag, 1); return 0; }
    f = (long long)d;
  }
  // x >= low, so the difference is exact in uint64
  const unsigned long long q = f < low ? 0ull : ((unsigned long long)f - (unsigned long long)low) / (unsigned)bw + 1;
  if (q < 1 || q > (unsigned long long)ng) { atomicOr(flag, 1); return 0; }
  return (int)q;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) texture_level_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                                 size_t n, int row, long long low, int bw, int ng,
                                                                 uint8_t* __restrict__ out, int* __restrict__ flag) {
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    unsigned w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (row == 256 ? l != 0 : l == row) w[k >> 2] |= (unsigned)level_of(vol[base + k], low, bw, ng, flag) << (8 * (k & 3));
    }
    const uint4 lv = make_uint4(w[0], w[1], w[2], w[3]);
    if (base + kChunk <= n) {
      reinterpret_cast<uint4*>(out)[c] = lv;
    } else {
      for (int k = 0; base + k < n; ++k) out[base + k] = (uint8_t)label_at(lv, k);
    }
  }
}

// ---- GLCM -----------------------------------------------------------------------------------------------------------
// Direction d: (0,0,1); (0,1,-1..1); (1,-1..1,-1..1), as (dz, dy, dx) over array axes (0, 1, 2).
__host__ __device__ constexpr int dir_z(int d) { return d < 4 ? 0 : 1; }
__host__ __device__ constexpr int dir_y(int d) { return d == 0 ? 0 : (d < 4 ? 1 : (d - 4) / 3 - 1); }
__host__ __device__ constexpr int dir_x(int d) { return d == 0 ? 1 : (d < 4 ? d - 2 : (d - 4) % 3 - 1); }

// (i, j), 1 <= i <= j <= ng -> row-major upper-triangle index
__host__ __device__ __forceinline__ int tri(int i, int j, int ng) { return (i - 1) * ng - (i - 1) * (i - 2) / 2 + (j - i); }

// kTri: shared counters s[d][tri(i, j)].  Otherwise s[d][(j - i) * ng + i - 1] for j - i < kBand, global for the rest.
template <bool kTri>
__global__ void __launch_bounds__(kThreads) glcm_kernel(const uint8_t* __restrict__ lev, int n0, int n1, int n2, int ng,
                                                        uint32_t* __restrict__ counts, int* __restrict__ flag) {
  extern __shared__ uint32_t s_cnt[];
  const int t_len = ng * (ng + 1) / 2;
  const int per_dir = kTri ? t_len : ng * kBand;
  for (int i = threadIdx.x; i < kGlcmDirections * per_dir; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int runs_x = (n2 + 31) / 32;
  const size_t runs = (size_t)n0 * n1 * runs_x;
  for (size_t r = warp; r < runs; r += n_warps) {   // warp-uniform
    const size_t line = r / runs_x;
    const int x = (int)(r % runs_x) * 32 + lane, y = (int)(line % n1), z = (int)(line / n1);
    const size_t v = line * n2 + x;
    int a = x < n2 ? lev[v] : 0;
    if (a > ng) { atomicOr(flag, 1); a = 0; }
    if (!__any_sync(kFull, a != 0)) continue;
#pragma unroll
    for (int d = 0; d < kGlcmDirections; ++d) {
      const int zz = z + dir_z(d), yy = y + dir_y(d), xx = x + dir_x(d);
      int b = 0;
      if (a && zz < n0 && (unsigned)yy < (unsigned)n1 && (unsigned)xx < (unsigned)n2)
        b = lev[(size_t)((long long)v + ((long long)dir_z(d) * n1 + dir_y(d)) * n2 + dir_x(d))];
      if (b > ng) { atomicOr(flag, 1); b = 0; }
      if (b) {
        const int i = min(a, b), j = max(a, b);
        const bool shared = kTri || j - i < kBand;
        const int key = kTri ? tri(i, j, ng) : (shared ? (j - i) * ng + i - 1 : per_dir + tri(i, j, ng));
        const unsigned peers = __match_any_sync(__activemask(), key);
        if (lane == __ffs(peers) - 1) {
          if (shared) atomicAdd(&s_cnt[d * per_dir + key], (uint32_t)__popc(peers));
          else atomicAdd(&counts[(size_t)d * t_len + (key - per_dir)], (uint32_t)__popc(peers));
        }
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kGlcmDirections * per_dir; k += blockDim.x) {
    if (!s_cnt[k]) continue;
    const int d = k / per_dir, e = k % per_dir;
    const int t = kTri ? e : tri(e % ng + 1, e % ng + 1 + e / ng, ng);
    atomicAdd(&counts[(size_t)d * t_len + t], s_cnt[k]);
  }
}

// ---- GLRLM ----------------------------------------------------------------------------------------------------------
// counts: global [13][ng][max_len] uint32 (a direction holds at most n runs).  Shared s[d][i - 1][len - 1] for
// len <= k_short; longer runs go straight to global.
__global__ void __launch_bounds__(kThreads) glrlm_kernel(const uint8_t* __restrict__ lev, int n0, int n1, int n2, int ng,
                                                         int max_len, int k_short, uint32_t* __restrict__ counts,
                                                         int* __restrict__ flag) {
  extern __shared__ uint32_t s_runs[];
  const int per_dir = ng * k_short;
  for (int i = threadIdx.x; i < kGlcmDirections * per_dir; i += blockDim.x) s_runs[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int runs_x = (n2 + 31) / 32;
  const size_t segs = (size_t)n0 * n1 * runs_x;
  for (size_t r = warp; r < segs; r += n_warps) {   // warp-uniform
    const size_t line = r / runs_x;
    const int x = (int)(r % runs_x) * 32 + lane, y = (int)(line % n1), z = (int)(line / n1);
    const size_t v = line * n2 + x;
    int a = x < n2 ? lev[v] : 0;
    if (a > ng) { atomicOr(flag, 1); a = 0; }
    if (!__any_sync(kFull, a != 0)) continue;
#pragma unroll 1
    for (int d = 0; d < kGlcmDirections; ++d) {
      const int dz = dir_z(d), dy = dir_y(d), dx = dir_x(d);
      const long long step = ((long long)dz * n1 + dy) * n2 + dx;
      int len = 0;
      if (a) {
        const int pz = z - dz, py = y - dy, px = x - dx;
        const bool continues = pz >= 0 && (unsigned)py < (unsigned)n1 && (unsigned)px < (unsigned)n2 &&
                               lev[(size_t)((long long)v - step)] == a;
        if (!continues) {   // v starts a run: walk to its end
          len = 1;
          int zz = z + dz, yy = y + dy, xx = x + dx;
          long long u = (long long)v + step;
          while (zz < n0 && (unsigned)yy < (unsigned)n1 && (unsigned)xx < (unsigned)n2 && lev[(size_t)u] == a) {
            ++len;
            zz += dz, yy += dy, xx += dx, u += step;
          }
        }
      }
      const unsigned long long key = len ? ((unsigned long long)len << 8) | (unsigned)a : 0ull;
      const unsigned peers = __match_any_sync(kFull, key);
      if (len && lane == __ffs(peers) - 1) {
        if (len <= k_short) atomicAdd(&s_runs[d * per_dir + (a - 1) * k_short + len - 1], (uint32_t)__popc(peers));
        else atomicAdd(&counts[((size_t)d * ng + a - 1) * max_len + len - 1], (uint32_t)__popc(peers));
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kGlcmDirections * per_dir; k += blockDim.x) {
    if (!s_runs[k]) continue;
    const int d = k / per_dir, e = k % per_dir;
    atomicAdd(&counts[((size_t)d * ng + e / k_short) * max_len + e % k_short], s_runs[k]);
  }
}

// ---- GLDM / NGTDM ---------------------------------------------------------------------------------------------------
// Per (level i, 0..26) cell: dependence G(i, c), count N(i, W), sum A(i, W).  Shared: the uint64 sums, then the two
// uint32 arrays, ng * 27 each (110,160 B at ng = 255).
__global__ void __launch_bounds__(kThreads) neighbour_kernel(const uint8_t* __restrict__ lev, int n0, int n1, int n2, int ng,
                                                             int alpha, uint32_t* __restrict__ dep, uint32_t* __restrict__ cnt,
                                                             unsigned long long* __restrict__ sums, int* __restrict__ flag) {
  extern __shared__ unsigned long long s_sum[];
  const int cells = ng * kNeighbourCells;
  uint32_t* s_dep = reinterpret_cast<uint32_t*>(s_sum + cells);
  uint32_t* s_cnt = s_dep + cells;
  for (int i = threadIdx.x; i < cells; i += blockDim.x) s_sum[i] = 0, s_dep[i] = 0, s_cnt[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int runs_x = (n2 + 31) / 32;
  const size_t segs = (size_t)n0 * n1 * runs_x;
  for (size_t r = warp; r < segs; r += n_warps) {   // warp-uniform
    const size_t line = r / runs_x;
    const int x = (int)(r % runs_x) * 32 + lane, y = (int)(line % n1), z = (int)(line / n1);
    const size_t v = line * n2 + x;
    int a = x < n2 ? lev[v] : 0;
    if (a > ng) { atomicOr(flag, 1); a = 0; }
    if (!__any_sync(kFull, a != 0)) continue;
    int w = 0, s = 0, c = 0;
    if (a) {
#pragma unroll
      for (int k = 0; k < 27; ++k) {
        if (k == 13) continue;   // the voxel itself
        const int dz = k / 9 - 1, dy = k / 3 % 3 - 1, dx = k % 3 - 1;
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        int b = 0;
        if ((unsigned)zz < (unsigned)n0 && (unsigned)yy < (unsigned)n1 && (unsigned)xx < (unsigned)n2)
          b = lev[(size_t)((long long)v + ((long long)dz * n1 + dy) * n2 + dx)];
        if (b > ng) b = 0;   // flagged by the lane that holds it
        if (b) {
          ++w;
          s += b;
          c += abs(b - a) <= alpha;
        }
      }
    }
    const int kd = a ? (a - 1) * kNeighbourCells + c : -1, kn = a ? (a - 1) * kNeighbourCells + w : -1;
    const unsigned pd = __match_any_sync(kFull, kd), pn = __match_any_sync(kFull, kn);
    const unsigned sum = __reduce_add_sync(pn, (unsigned)abs(w * a - s));   // < 32 * 2^13 over a peer group
    if (a && lane == __ffs(pd) - 1) atomicAdd(&s_dep[kd], (uint32_t)__popc(pd));
    if (a && lane == __ffs(pn) - 1) {
      atomicAdd(&s_cnt[kn], (uint32_t)__popc(pn));
      if (sum) atomicAdd(&s_sum[kn], (unsigned long long)sum);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < cells; k += blockDim.x) {
    if (s_dep[k]) atomicAdd(&dep[k], s_dep[k]);
    if (s_cnt[k]) atomicAdd(&cnt[k], s_cnt[k]);
    if (s_sum[k]) atomicAdd(&sums[k], s_sum[k]);
  }
}

// ---- generalised neighbourhoods (DESIGN §4.18) ----------------------------------------------------------------------
// An offset list travels as a kernel parameter (constant bank): offset k packs (dz, dy, dx) as three signed bytes.
struct OffsetList {
  int o[kMaxOffsets];
};
__device__ __forceinline__ int off_z(int p) { return (int)(signed char)(p & 0xff); }
__device__ __forceinline__ int off_y(int p) { return (int)(signed char)((p >> 8) & 0xff); }
__device__ __forceinline__ int off_x(int p) { return (int)(signed char)((p >> 16) & 0xff); }

// glcm_kernel over the offsets first .. first + count - 1 of `offs`: the same warp layout, key aggregation and shared
// layout (kTri: the triangle of every offset of the group; otherwise the band j - i < kBand, the rest global).
template <bool kTri>
__global__ void __launch_bounds__(kThreads) glcm_offsets_kernel(const uint8_t* __restrict__ lev, int n0, int n1, int n2, int ng,
                                                                OffsetList offs, int first, int count,
                                                                uint32_t* __restrict__ counts, int* __restrict__ flag) {
  extern __shared__ uint32_t s_cnt[];
  const int t_len = ng * (ng + 1) / 2;
  const int per_dir = kTri ? t_len : ng * kBand;
  for (int i = threadIdx.x; i < count * per_dir; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int runs_x = (n2 + 31) / 32;
  const size_t runs = (size_t)n0 * n1 * runs_x;
  for (size_t r = warp; r < runs; r += n_warps) {   // warp-uniform
    const size_t line = r / runs_x;
    const int x = (int)(r % runs_x) * 32 + lane, y = (int)(line % n1), z = (int)(line / n1);
    const size_t v = line * n2 + x;
    int a = x < n2 ? lev[v] : 0;
    if (a > ng) { atomicOr(flag, 1); a = 0; }
    if (!__any_sync(kFull, a != 0)) continue;
#pragma unroll 1
    for (int d = 0; d < count; ++d) {
      const int p = offs.o[first + d], dz = off_z(p), dy = off_y(p), dx = off_x(p);
      const int zz = z + dz, yy = y + dy, xx = x + dx;
      int b = 0;
      if (a && (unsigned)zz < (unsigned)n0 && (unsigned)yy < (unsigned)n1 && (unsigned)xx < (unsigned)n2)
        b = lev[(size_t)((long long)v + ((long long)dz * n1 + dy) * n2 + dx)];
      if (b > ng) { atomicOr(flag, 1); b = 0; }
      if (b) {
        const int i = min(a, b), j = max(a, b);
        const bool shared = kTri || j - i < kBand;
        const int key = kTri ? tri(i, j, ng) : (shared ? (j - i) * ng + i - 1 : per_dir + tri(i, j, ng));
        const unsigned peers = __match_any_sync(__activemask(), key);
        if (lane == __ffs(peers) - 1) {
          if (shared) atomicAdd(&s_cnt[d * per_dir + key], (uint32_t)__popc(peers));
          else atomicAdd(&counts[(size_t)(first + d) * t_len + (key - per_dir)], (uint32_t)__popc(peers));
        }
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < count * per_dir; k += blockDim.x) {
    if (!s_cnt[k]) continue;
    const int d = k / per_dir, e = k % per_dir;
    const int t = kTri ? e : tri(e % ng + 1, e % ng + 1 + e / ng, ng);
    atomicAdd(&counts[(size_t)(first + d) * t_len + t], s_cnt[k]);
  }
}

// neighbour_kernel over the neighbourhood +-offs (K = 2 n neighbours, cols = K + 1 cells per level).  kShared: the
// counters of every level in shared memory (ng * cols * 16 B); otherwise warp-aggregated global atomics.  Warp sums of
// |W i - S| < 32 * 342 * 254 < 2^22 fit in 32 bits.
template <bool kShared>
__global__ void __launch_bounds__(kThreads) neighbour_offsets_kernel(const uint8_t* __restrict__ lev, int n0, int n1, int n2,
                                                                     int ng, int alpha, OffsetList offs, int n_offs, int cols,
                                                                     uint32_t* __restrict__ dep, uint32_t* __restrict__ cnt,
                                                                     unsigned long long* __restrict__ sums,
                                                                     int* __restrict__ flag) {
  extern __shared__ unsigned long long s_sum[];
  const int cells = ng * cols;
  uint32_t* s_dep = reinterpret_cast<uint32_t*>(s_sum + cells);
  uint32_t* s_cnt = s_dep + cells;
  if (kShared) {
    for (int i = threadIdx.x; i < cells; i += blockDim.x) s_sum[i] = 0, s_dep[i] = 0, s_cnt[i] = 0;
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int runs_x = (n2 + 31) / 32;
  const size_t segs = (size_t)n0 * n1 * runs_x;
  for (size_t r = warp; r < segs; r += n_warps) {   // warp-uniform
    const size_t line = r / runs_x;
    const int x = (int)(r % runs_x) * 32 + lane, y = (int)(line % n1), z = (int)(line / n1);
    const size_t v = line * n2 + x;
    int a = x < n2 ? lev[v] : 0;
    if (a > ng) { atomicOr(flag, 1); a = 0; }
    if (!__any_sync(kFull, a != 0)) continue;
    int w = 0, s = 0, c = 0;
    if (a) {
#pragma unroll 1
      for (int k = 0; k < n_offs; ++k) {
        const int p = offs.o[k], dz = off_z(p), dy = off_y(p), dx = off_x(p);
        const long long step = ((long long)dz * n1 + dy) * n2 + dx;
#pragma unroll
        for (int sgn = 1; sgn >= -1; sgn -= 2) {
          const int zz = z + sgn * dz, yy = y + sgn * dy, xx = x + sgn * dx;
          int b = 0;
          if ((unsigned)zz < (unsigned)n0 && (unsigned)yy < (unsigned)n1 && (unsigned)xx < (unsigned)n2)
            b = lev[(size_t)((long long)v + sgn * step)];
          if (b > ng) b = 0;   // flagged by the lane that holds it
          if (b) {
            ++w;
            s += b;
            c += abs(b - a) <= alpha;
          }
        }
      }
    }
    const int kd = a ? (a - 1) * cols + c : -1, kn = a ? (a - 1) * cols + w : -1;
    const unsigned pd = __match_any_sync(kFull, kd), pn = __match_any_sync(kFull, kn);
    const unsigned sum = __reduce_add_sync(pn, (unsigned)abs(w * a - s));
    if (a && lane == __ffs(pd) - 1) atomicAdd(kShared ? &s_dep[kd] : &dep[kd], (uint32_t)__popc(pd));
    if (a && lane == __ffs(pn) - 1) {
      atomicAdd(kShared ? &s_cnt[kn] : &cnt[kn], (uint32_t)__popc(pn));
      if (sum) atomicAdd(kShared ? &s_sum[kn] : &sums[kn], (unsigned long long)sum);
    }
  }
  if (kShared) {
    __syncthreads();
    for (int k = threadIdx.x; k < cells; k += blockDim.x) {
      if (s_dep[k]) atomicAdd(&dep[k], s_dep[k]);
      if (s_cnt[k]) atomicAdd(&cnt[k], s_cnt[k]);
      if (s_sum[k]) atomicAdd(&sums[k], s_sum[k]);
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// The work area: the flag, then the pair counts.
size_t work_bytes(int n_levels) {
  return align256(sizeof(int)) + align256((size_t)kGlcmDirections * n_levels * (n_levels + 1) / 2 * 4);
}

template <typename K>
int grid_for(K kernel, size_t smem, size_t work, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (work + kThreads - 1) / kThreads;
  return (int)std::max<size_t>(std::min((size_t)per_sm * num_sms, need), 1);
}

template <typename T>
int launch_levels(const void* vol, const uint8_t* mask, size_t n, int row, long long low, int bw, int ng, uint8_t* out,
                  int* flag, int num_sms, cudaStream_t st) {
  const size_t chunks = (n + kChunk - 1) / kChunk;
  texture_level_kernel<T><<<grid_for(texture_level_kernel<T>, 0, chunks, num_sms), kThreads, 0, st>>>(
      static_cast<const T*>(vol), mask, n, row, low, bw, ng, out, flag);
  return (int)cudaGetLastError();
}

int flag_result(const int* d_flag, cudaStream_t st) {
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return (flag & 2) ? kLevelNonFinite : ((flag & 1) ? kLevelRange : 0);
}

}  // namespace

int TextureWork::reserve(size_t bytes) {
  if (bytes <= d_bytes) return 0;
  release();
  const cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) { d = nullptr; return (int)e; }
  d_bytes = bytes;
  return 0;
}

void TextureWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  d_bytes = 0;
}

int texture_levels(TextureWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, size_t n, int row, int64_t low,
                   int bin_width, int n_levels, uint8_t* d_levels, int num_sms, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve(work_bytes(1)));
  int* flag = static_cast<int*>(w.d);
  SC(cudaMemsetAsync(flag, 0, sizeof(int), st));
  int rc;
#define LM_LEVELS_CASE(code, T) \
  case code: rc = launch_levels<T>(d_vol, d_mask, n, row, low, bin_width, n_levels, d_levels, flag, num_sms, st); break
  switch (dtype) {
    LM_LEVELS_CASE(LM_DTYPE_U8, uint8_t);
    LM_LEVELS_CASE(LM_DTYPE_I8, int8_t);
    LM_LEVELS_CASE(LM_DTYPE_I16, int16_t);
    LM_LEVELS_CASE(LM_DTYPE_I32, int32_t);
    LM_LEVELS_CASE(LM_DTYPE_I64, int64_t);
    LM_LEVELS_CASE(LM_DTYPE_F16, __half);
    LM_LEVELS_CASE(LM_DTYPE_BF16, __nv_bfloat16);
    LM_LEVELS_CASE(LM_DTYPE_F32, float);
    LM_LEVELS_CASE(LM_DTYPE_F64, double);
    default: return -1;
  }
#undef LM_LEVELS_CASE
  if (rc) return rc;
  ++*launches;
  return flag_result(flag, st);
}

int glcm(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, int num_sms,
         cudaStream_t st, int64_t* launches) {
  const size_t t_len = (size_t)n_levels * (n_levels + 1) / 2, total = kGlcmDirections * t_len;
  SC((cudaError_t)w.reserve(work_bytes(n_levels)));
  int* flag = static_cast<int*>(w.d);
  uint32_t* d_counts = reinterpret_cast<uint32_t*>(static_cast<char*>(w.d) + align256(sizeof(int)));
  SC(cudaMemsetAsync(flag, 0, sizeof(int), st));
  SC(cudaMemsetAsync(d_counts, 0, total * 4, st));
  const size_t runs = (size_t)n0 * n1 * ((n2 + 31) / 32), threads = runs * 32;
  if (n_levels <= kSmemLevels) {
    const size_t smem = total * 4;
    SC(cudaFuncSetAttribute(glcm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    glcm_kernel<true><<<grid_for(glcm_kernel<true>, smem, threads, num_sms), kThreads, smem, st>>>(d_levels, n0, n1, n2, n_levels,
                                                                                                   d_counts, flag);
  } else {
    const size_t smem = (size_t)kGlcmDirections * n_levels * kBand * 4;
    SC(cudaFuncSetAttribute(glcm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    glcm_kernel<false><<<grid_for(glcm_kernel<false>, smem, threads, num_sms), kThreads, smem, st>>>(d_levels, n0, n1, n2,
                                                                                                     n_levels, d_counts, flag);
  }
  SC(cudaGetLastError());
  ++*launches;
  std::vector<uint32_t> h(total);
  SC(cudaMemcpyAsync(h.data(), d_counts, total * 4, cudaMemcpyDeviceToHost, st));
  const int rc = flag_result(flag, st);
  if (rc) return rc;
  for (size_t k = 0; k < total; ++k) counts[k] = h[k];
  return 0;
}

int glrlm(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, int num_sms,
          cudaStream_t st, int64_t* launches) {
  const int max_len = std::max(n0, std::max(n1, n2));
  const int k_short = std::min(kSmemWords / (kGlcmDirections * n_levels), max_len);
  const size_t total = (size_t)kGlcmDirections * n_levels * max_len;
  SC((cudaError_t)w.reserve(align256(sizeof(int)) + align256(total * 4)));
  int* flag = static_cast<int*>(w.d);
  uint32_t* d_counts = reinterpret_cast<uint32_t*>(static_cast<char*>(w.d) + align256(sizeof(int)));
  SC(cudaMemsetAsync(flag, 0, sizeof(int), st));
  SC(cudaMemsetAsync(d_counts, 0, total * 4, st));
  const size_t threads = (size_t)n0 * n1 * ((n2 + 31) / 32) * 32;
  const size_t smem = (size_t)kGlcmDirections * n_levels * k_short * 4;
  SC(cudaFuncSetAttribute(glrlm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  glrlm_kernel<<<grid_for(glrlm_kernel, smem, threads, num_sms), kThreads, smem, st>>>(d_levels, n0, n1, n2, n_levels, max_len,
                                                                                      k_short, d_counts, flag);
  SC(cudaGetLastError());
  ++*launches;
  std::vector<uint32_t> h(total);
  SC(cudaMemcpyAsync(h.data(), d_counts, total * 4, cudaMemcpyDeviceToHost, st));
  const int rc = flag_result(flag, st);
  if (rc) return rc;
  for (size_t k = 0; k < total; ++k) counts[k] = h[k];
  return 0;
}

int neighbour_counts(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                     int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums, int num_sms, cudaStream_t st,
                     int64_t* launches) {
  const size_t cells = (size_t)n_levels * kNeighbourCells;
  const size_t sums_at = align256(sizeof(int)), dep_at = sums_at + align256(cells * 8), cnt_at = dep_at + align256(cells * 4);
  SC((cudaError_t)w.reserve(cnt_at + align256(cells * 4)));
  char* base = static_cast<char*>(w.d);
  int* flag = reinterpret_cast<int*>(base);
  unsigned long long* d_sums = reinterpret_cast<unsigned long long*>(base + sums_at);
  uint32_t* d_dep = reinterpret_cast<uint32_t*>(base + dep_at);
  uint32_t* d_cnt = reinterpret_cast<uint32_t*>(base + cnt_at);
  SC(cudaMemsetAsync(base, 0, cnt_at + cells * 4, st));
  const size_t threads = (size_t)n0 * n1 * ((n2 + 31) / 32) * 32;
  const size_t smem = cells * 16;
  SC(cudaFuncSetAttribute(neighbour_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  neighbour_kernel<<<grid_for(neighbour_kernel, smem, threads, num_sms), kThreads, smem, st>>>(d_levels, n0, n1, n2, n_levels,
                                                                                              alpha, d_dep, d_cnt, d_sums, flag);
  SC(cudaGetLastError());
  ++*launches;
  std::vector<unsigned long long> hs(cells);
  std::vector<uint32_t> hd(cells), hc(cells);
  SC(cudaMemcpyAsync(hs.data(), d_sums, cells * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(hd.data(), d_dep, cells * 4, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(hc.data(), d_cnt, cells * 4, cudaMemcpyDeviceToHost, st));
  const int rc = flag_result(flag, st);
  if (rc) return rc;
  for (size_t k = 0; k < cells; ++k) dependence[k] = hd[k], ngtdm_counts[k] = hc[k], ngtdm_sums[k] = (int64_t)hs[k];
  return 0;
}

namespace {
OffsetList pack_offsets(const int8_t* offsets, int n) {
  OffsetList l{};
  for (int k = 0; k < n; ++k)
    l.o[k] = (int)(uint8_t)offsets[3 * k] | ((int)(uint8_t)offsets[3 * k + 1] << 8) | ((int)(uint8_t)offsets[3 * k + 2] << 16);
  return l;
}
}  // namespace

int glcm_offsets(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, const int8_t* offsets,
                 int n_offsets, int64_t* counts, int num_sms, cudaStream_t st, int64_t* launches) {
  const size_t t_len = (size_t)n_levels * (n_levels + 1) / 2, total = (size_t)n_offsets * t_len;
  SC((cudaError_t)w.reserve(align256(sizeof(int)) + align256(total * 4)));
  int* flag = static_cast<int*>(w.d);
  uint32_t* d_counts = reinterpret_cast<uint32_t*>(static_cast<char*>(w.d) + align256(sizeof(int)));
  SC(cudaMemsetAsync(flag, 0, sizeof(int), st));
  SC(cudaMemsetAsync(d_counts, 0, total * 4, st));
  const OffsetList offs = pack_offsets(offsets, n_offsets);
  const size_t threads = (size_t)n0 * n1 * ((n2 + 31) / 32) * 32;
  const bool tri_layout = n_levels <= kSmemLevels;
  const int per_dir = tri_layout ? (int)t_len : n_levels * kBand;
  const int group = std::max(1, std::min(n_offsets, kSmemWords / per_dir));   // >= 13: per_dir <= 4095
  for (int first = 0; first < n_offsets; first += group) {
    const int count = std::min(group, n_offsets - first);
    const size_t smem = (size_t)count * per_dir * 4;
    if (tri_layout) {
      SC(cudaFuncSetAttribute(glcm_offsets_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      glcm_offsets_kernel<true><<<grid_for(glcm_offsets_kernel<true>, smem, threads, num_sms), kThreads, smem, st>>>(
          d_levels, n0, n1, n2, n_levels, offs, first, count, d_counts, flag);
    } else {
      SC(cudaFuncSetAttribute(glcm_offsets_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      glcm_offsets_kernel<false><<<grid_for(glcm_offsets_kernel<false>, smem, threads, num_sms), kThreads, smem, st>>>(
          d_levels, n0, n1, n2, n_levels, offs, first, count, d_counts, flag);
    }
    SC(cudaGetLastError());
    ++*launches;
  }
  std::vector<uint32_t> h(total);
  SC(cudaMemcpyAsync(h.data(), d_counts, total * 4, cudaMemcpyDeviceToHost, st));
  const int rc = flag_result(flag, st);
  if (rc) return rc;
  for (size_t k = 0; k < total; ++k) counts[k] = h[k];
  return 0;
}

int neighbour_offsets(TextureWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                      const int8_t* offsets, int n_offsets, int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums,
                      int num_sms, cudaStream_t st, int64_t* launches) {
  const int cols = 2 * n_offsets + 1;
  const size_t cells = (size_t)n_levels * cols;
  const size_t sums_at = align256(sizeof(int)), dep_at = sums_at + align256(cells * 8), cnt_at = dep_at + align256(cells * 4);
  SC((cudaError_t)w.reserve(cnt_at + align256(cells * 4)));
  char* base = static_cast<char*>(w.d);
  int* flag = reinterpret_cast<int*>(base);
  unsigned long long* d_sums = reinterpret_cast<unsigned long long*>(base + sums_at);
  uint32_t* d_dep = reinterpret_cast<uint32_t*>(base + dep_at);
  uint32_t* d_cnt = reinterpret_cast<uint32_t*>(base + cnt_at);
  SC(cudaMemsetAsync(base, 0, cnt_at + cells * 4, st));
  const OffsetList offs = pack_offsets(offsets, n_offsets);
  const size_t threads = (size_t)n0 * n1 * ((n2 + 31) / 32) * 32;
  if (cells * 16 <= (size_t)kSmemWords * 4) {
    const size_t smem = cells * 16;
    SC(cudaFuncSetAttribute(neighbour_offsets_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    neighbour_offsets_kernel<true><<<grid_for(neighbour_offsets_kernel<true>, smem, threads, num_sms), kThreads, smem, st>>>(
        d_levels, n0, n1, n2, n_levels, alpha, offs, n_offsets, cols, d_dep, d_cnt, d_sums, flag);
  } else {
    neighbour_offsets_kernel<false><<<grid_for(neighbour_offsets_kernel<false>, 0, threads, num_sms), kThreads, 0, st>>>(
        d_levels, n0, n1, n2, n_levels, alpha, offs, n_offsets, cols, d_dep, d_cnt, d_sums, flag);
  }
  SC(cudaGetLastError());
  ++*launches;
  std::vector<unsigned long long> hs(cells);
  std::vector<uint32_t> hd(cells), hc(cells);
  SC(cudaMemcpyAsync(hs.data(), d_sums, cells * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(hd.data(), d_dep, cells * 4, cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(hc.data(), d_cnt, cells * 4, cudaMemcpyDeviceToHost, st));
  const int rc = flag_result(flag, st);
  if (rc) return rc;
  for (size_t k = 0; k < cells; ++k) dependence[k] = hd[k], ngtdm_counts[k] = hc[k], ngtdm_sums[k] = (int64_t)hs[k];
  return 0;
}

}  // namespace lm
