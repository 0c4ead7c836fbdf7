// Regional lung statistics support (lm_plane_label_counts_dev, lm_surface_distance_dev, lm_region_map_dev; DESIGN §4.8).
//
// Plane counts: a thread owns one axis-2 position x (a warp's lanes take 32 adjacent x) and walks kPlaneRun voxels along
// a line that stays inside one plane of the counted axis (axis 1 for planes of axes 0 and 2, axis 0 for planes of axis 1).
// It counts the run of its current label and adds it to the global [plane][257] table only when the label changes, so a
// lung interior costs two 64-bit atomics per kPlaneRun voxels.  Label 0 is not counted: the host derives it from the
// union column.
//
// Surface distance: an exact Euclidean distance transform in three separable passes, squared distances in float64.
//   A. along axis 2: one warp per row, a max-scan of the background positions from the left and a min-scan from the right
//      give each voxel its nearest background voxel in the row; d2 = (dx * s2)^2, +inf for a row without background.
//   B. along axis 1, C. along axis 0: one thread per line, lanes on adjacent x (coalesced); the lower envelope of the
//      parabolas f(j) + ((q - j) * s)^2 over the finite f(j) (Felzenszwalb & Huttenlocher, Theory of Computing 8, 2012).
//      The envelope's stacks (vertex, f) live in the work area, entry k of line L at k * n_lines + L, so they are coalesced
//      too and any line length works.  The evaluation walks the envelope by comparing the float64 values of consecutive
//      parabolas rather than their rounded intersections, so it returns the minimum over the envelope exactly.
//   C writes float32(sqrt(d2)) to the caller's output.
// Region map: 16 mask bytes per thread (mask_chunk.cuh); map = lut[bucket * 256 + label], bucket = plane index along an
// axis or the number of shell bounds <= distance.
#include <math.h>

#include <algorithm>

#include "mask_chunk.cuh"
#include "regions.cuh"

namespace lm {
namespace {

constexpr int kThreads = 256;
constexpr int kPlaneRun = 64;   // voxels one plane-count thread walks
constexpr int kMaxBounds = 255;

typedef unsigned long long u64;

// ---- plane counts ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) plane_count_kernel(const uint8_t* __restrict__ mask, int n0, int n1, int n2, int axis,
                                                               u64* __restrict__ counts) {
  const int n_walk = axis == 1 ? n0 : n1, n_fix = axis == 1 ? n1 : n0;
  const size_t walk_stride = axis == 1 ? (size_t)n1 * n2 : (size_t)n2, fix_stride = axis == 1 ? (size_t)n2 : (size_t)n1 * n2;
  const size_t x_tiles = (n2 + 31) / 32, stripes = (n_walk + kPlaneRun - 1) / kPlaneRun;
  const size_t items = (size_t)n_fix * stripes * x_tiles * 32;
  for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < items; j += (size_t)gridDim.x * blockDim.x) {
    size_t r = j >> 5;
    const int x = (int)(r % x_tiles) * 32 + (int)(j & 31);
    r /= x_tiles;
    const int s = (int)(r % stripes), f = (int)(r / stripes);
    if (x >= n2) continue;
    const size_t plane = axis == 2 ? (size_t)x : (size_t)f;
    const int w0 = s * kPlaneRun, w1 = min(n_walk, w0 + kPlaneRun);
    const uint8_t* p = mask + f * fix_stride + (size_t)w0 * walk_stride + x;
    u64* row = counts + plane * kPlaneRows;
    int cur = 0;
    unsigned run = 0, any = 0;
    for (int w = w0; w < w1; ++w, p += walk_stride) {
      const int l = __ldg(p);
      any += l != 0;
      if (l != cur) {
        if (cur && run) atomicAdd(&row[cur], (u64)run);
        cur = l;
        run = 0;
      }
      ++run;
    }
    if (cur && run) atomicAdd(&row[cur], (u64)run);
    if (any) atomicAdd(&row[kPlaneRows - 1], (u64)any);
  }
}

// ---- distance transform ------------------------------------------------------------------------------------------------
// A: one warp per row of n2 voxels.  The left scan parks the nearest background position at or left of x in d2 (exact as a
// double); the right scan reads it back in the same lane.
__global__ void __launch_bounds__(kThreads) edt_rows_kernel(const uint8_t* __restrict__ mask, size_t rows, int n2, double s2,
                                                            double* __restrict__ d2) {
  const int lane = threadIdx.x & 31;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  constexpr int kNone = 0x7FFFFFFF;
  for (size_t row = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const uint8_t* m = mask + row * n2;
    double* o = d2 + row * n2;
    int carry = -1;
    for (int x0 = 0; x0 < n2; x0 += 32) {
      const int x = x0 + lane;
      int z = (x < n2 && __ldg(m + x) == 0) ? x : -1;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) z = max(z, __shfl_up_sync(0xFFFFFFFFu, z, off));
      z = max(z, carry);
      carry = __shfl_sync(0xFFFFFFFFu, z, 31);
      if (x < n2) o[x] = (double)z;
    }
    carry = kNone;
    for (int x0 = (n2 - 1) / 32 * 32; x0 >= 0; x0 -= 32) {
      const int x = x0 + lane;
      int z = (x < n2 && __ldg(m + x) == 0) ? x : kNone;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) z = min(z, __shfl_down_sync(0xFFFFFFFFu, z, off));
      z = min(z, carry);
      carry = __shfl_sync(0xFFFFFFFFu, z, 0);
      if (x < n2) {
        const int left = (int)o[x];
        const int d = min(left >= 0 ? x - left : kNone, z != kNone ? z - x : kNone);
        const double dd = (double)d * s2;
        o[x] = d == kNone ? (double)INFINITY : dd * dd;
      }
    }
  }
}

// Abscissa where the parabolas of vertices a < b (weight w = s^2) meet.
__device__ __forceinline__ double meet(int a, double fa, int b, double fb, double w) {
  return ((fb + w * ((double)b * b)) - (fa + w * ((double)a * a))) / (2.0 * w * (double)(b - a));
}

// B / C: line L holds the len voxels base + j * inner, base = (L / inner) * len * inner + L % inner.  kFinal: read d2, write
// float32 sqrt to out; otherwise in place on d2.
template <bool kFinal>
__global__ void __launch_bounds__(kThreads) edt_lines_kernel(double* __restrict__ d2, float* __restrict__ out, size_t lines,
                                                             int len, size_t inner, double s, int* __restrict__ sv,
                                                             double* __restrict__ sf) {
  const double w = s * s;
  for (size_t L = blockIdx.x * (size_t)blockDim.x + threadIdx.x; L < lines; L += (size_t)gridDim.x * blockDim.x) {
    const size_t base = (L / inner) * (size_t)len * inner + L % inner;
    // lower envelope: top of the stack in registers, the stack in sv / sf
    int k = -1, vk = 0;
    double fk = 0.0, zk = -INFINITY;
    double f_next = d2[base];
    for (int q = 0; q < len; ++q) {
      const double fq = f_next;
      if (q + 1 < len) f_next = d2[base + (size_t)(q + 1) * inner];
      if (!(fq < INFINITY)) continue;
      while (k >= 0 && meet(vk, fk, q, fq, w) <= zk) {
        --k;
        vk = sv[(size_t)k * lines + L];
        fk = sf[(size_t)k * lines + L];
        zk = k > 0 ? meet(sv[(size_t)(k - 1) * lines + L], sf[(size_t)(k - 1) * lines + L], vk, fk, w) : -INFINITY;
      }
      zk = k >= 0 ? meet(vk, fk, q, fq, w) : -INFINITY;
      ++k;
      sv[(size_t)k * lines + L] = vk = q;
      sf[(size_t)k * lines + L] = fk = fq;
    }
    const int top = k;
    int j = 0, vj = 0, vn = 0;
    double fj = INFINITY, fn = INFINITY;
    if (top >= 0) { vj = sv[L]; fj = sf[L]; }
    if (top >= 1) { vn = sv[lines + L]; fn = sf[lines + L]; }
    for (int q = 0; q < len; ++q) {
      double cur = INFINITY;
      if (top >= 0) {
        const double dj = (double)(q - vj) * s;
        cur = fj + dj * dj;
        while (j < top) {
          const double dn = (double)(q - vn) * s, next = fn + dn * dn;
          if (next > cur) break;
          ++j;
          vj = vn; fj = fn; cur = next;
          if (j < top) { vn = sv[(size_t)(j + 1) * lines + L]; fn = sf[(size_t)(j + 1) * lines + L]; }
        }
      }
      if constexpr (kFinal) out[base + (size_t)q * inner] = (float)sqrt(cur);
      else d2[base + (size_t)q * inner] = cur;
    }
  }
}

// ---- region map ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) region_map_kernel(const uint8_t* __restrict__ mask, const float* __restrict__ dist,
                                                              size_t n, int n1, int n2, int axis, const float* __restrict__ bounds,
                                                              int n_bounds, const uint8_t* __restrict__ lut,
                                                              uint8_t* __restrict__ map) {
  __shared__ float s_bounds[kMaxBounds];
  for (int i = threadIdx.x; i < n_bounds; i += blockDim.x) s_bounds[i] = bounds[i];
  __syncthreads();
  const size_t chunks = (n + kChunk - 1) / kChunk;
  const bool vec_out = (reinterpret_cast<uintptr_t>(map) & 15) == 0;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    // coordinates of the chunk's first voxel, then stepped voxel by voxel
    const size_t row = base / (size_t)n2;
    int x = (int)(base - row * n2), p1 = (int)(row % (size_t)n1);
    size_t p0 = row / (size_t)n1;
    unsigned wv[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (l) {
        size_t b;
        if (dist) {
          const float d = dist[base + k];
          int m = 0;
          for (int i = 0; i < n_bounds; ++i) m += s_bounds[i] <= d;
          b = (size_t)m;
        } else {
          b = axis == 0 ? p0 : (size_t)(axis == 1 ? p1 : x);
        }
        wv[k >> 2] |= (unsigned)__ldg(lut + b * 256 + l) << (8 * (k & 3));
      }
      if (++x == n2) {
        x = 0;
        if (++p1 == n1) { p1 = 0; ++p0; }
      }
    }
    const uint4 codes = make_uint4(wv[0], wv[1], wv[2], wv[3]);
    if (vec_out && base + kChunk <= n) {
      reinterpret_cast<uint4*>(map)[c] = codes;
    } else {
      for (int k = 0; k < kChunk && base + k < n; ++k) map[base + k] = (uint8_t)label_at(codes, k);
    }
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------------
#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

template <typename K>
int grid_for(K kernel, size_t work, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (work + kThreads - 1) / kThreads;
  return (int)std::max<size_t>(std::min((size_t)per_sm * num_sms, need), 1);
}

}  // namespace

int RegionWork::reserve(size_t bytes) {
  if (bytes <= d_bytes) return 0;
  release();
  const cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) { d = nullptr; return (int)e; }
  d_bytes = bytes;
  return 0;
}

void RegionWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  d_bytes = 0;
}

int plane_label_counts(RegionWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int axis, int64_t* counts, int num_sms,
                       cudaStream_t st, int64_t* launches) {
  const int n_axis = axis == 0 ? n0 : (axis == 1 ? n1 : n2);
  const size_t bytes = (size_t)n_axis * kPlaneRows * sizeof(u64);
  SC((cudaError_t)w.reserve(bytes));
  u64* d_counts = static_cast<u64*>(w.d);
  SC(cudaMemsetAsync(d_counts, 0, bytes, st));
  const int n_walk = axis == 1 ? n0 : n1, n_fix = axis == 1 ? n1 : n0;
  const size_t items = (size_t)n_fix * ((n_walk + kPlaneRun - 1) / kPlaneRun) * ((n2 + 31) / 32) * 32;
  plane_count_kernel<<<grid_for(plane_count_kernel, items, num_sms), kThreads, 0, st>>>(d_mask, n0, n1, n2, axis, d_counts);
  SC(cudaGetLastError());
  ++*launches;
  SC(cudaMemcpyAsync(counts, d_counts, bytes, cudaMemcpyDeviceToHost, st));   // u64 counts below 2^63: int64 as they are
  SC(cudaStreamSynchronize(st));
  // the kernel skips label 0; a plane holds n / n_axis voxels
  const int64_t plane = (int64_t)n0 * n1 * n2 / n_axis;
  for (int p = 0; p < n_axis; ++p) counts[(size_t)p * kPlaneRows] = plane - counts[(size_t)p * kPlaneRows + kPlaneRows - 1];
  return 0;
}

int surface_distance(RegionWork& w, const uint8_t* d_mask, int n0, int n1, int n2, const double* spacing, float* d_out,
                     int num_sms, cudaStream_t st, int64_t* launches) {
  const size_t n = (size_t)n0 * n1 * n2;
  const size_t d2_bytes = align256(n * 8), sv_bytes = align256(n * 4);
  SC((cudaError_t)w.reserve(d2_bytes + sv_bytes + n * 8));
  double* d2 = static_cast<double*>(w.d);
  int* sv = reinterpret_cast<int*>(static_cast<char*>(w.d) + d2_bytes);
  double* sf = reinterpret_cast<double*>(static_cast<char*>(w.d) + d2_bytes + sv_bytes);

  const size_t rows = (size_t)n0 * n1;
  edt_rows_kernel<<<grid_for(edt_rows_kernel, rows * 32, num_sms), kThreads, 0, st>>>(d_mask, rows, n2, spacing[2], d2);
  const size_t lines1 = (size_t)n0 * n2, lines0 = (size_t)n1 * n2;
  edt_lines_kernel<false><<<grid_for(edt_lines_kernel<false>, lines1, num_sms), kThreads, 0, st>>>(
      d2, nullptr, lines1, n1, (size_t)n2, spacing[1], sv, sf);
  edt_lines_kernel<true><<<grid_for(edt_lines_kernel<true>, lines0, num_sms), kThreads, 0, st>>>(
      d2, d_out, lines0, n0, (size_t)n1 * n2, spacing[0], sv, sf);
  SC(cudaGetLastError());
  *launches += 3;
  return 0;
}

int region_map(RegionWork& w, const uint8_t* d_mask, const float* d_dist, int n0, int n1, int n2, int axis, const float* bounds,
               int n_bounds, const uint8_t* lut, size_t lut_size, uint8_t* d_map, int num_sms, cudaStream_t st,
               int64_t* launches) {
  const size_t n = (size_t)n0 * n1 * n2, bounds_at = align256(lut_size);
  SC((cudaError_t)w.reserve(bounds_at + kMaxBounds * sizeof(float)));
  uint8_t* d_lut = static_cast<uint8_t*>(w.d);
  float* d_bounds = reinterpret_cast<float*>(d_lut + bounds_at);
  SC(cudaMemcpyAsync(d_lut, lut, lut_size, cudaMemcpyHostToDevice, st));
  if (n_bounds) SC(cudaMemcpyAsync(d_bounds, bounds, n_bounds * sizeof(float), cudaMemcpyHostToDevice, st));
  const size_t chunks = (n + kChunk - 1) / kChunk;
  region_map_kernel<<<grid_for(region_map_kernel, chunks, num_sms), kThreads, 0, st>>>(
      d_mask, d_dist, n, n1, n2, axis, d_bounds, d_dist ? n_bounds : 0, d_lut, d_map);
  SC(cudaGetLastError());
  ++*launches;
  SC(cudaStreamSynchronize(st));   // the LUT and bounds are pageable host memory of the caller
  return 0;
}

}  // namespace lm
