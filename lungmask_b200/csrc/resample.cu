// PyRadiomics' resampling with the cubic B-spline or nearest-neighbour interpolator (lm_bspline_coefficients_dev,
// lm_resample_dev; DESIGN §4.19).
//
// The B-spline coefficients are the image's 1-D decompositions along x, then y, then z (Unser / Thevenaz, mirror
// boundaries, one pole z = sqrt(3) - 2), each line: times the gain; c[0] = the causal sum over the first 18 samples (lines
// of 19 or more) or the full mirror sum (shorter lines); c[n] += z c[n-1]; c[N-1] = anti (z c[N-2] + c[N-1]);
// c[n] = z (c[n+1] - c[n]).  A line of one voxel is left unchanged.  The recursion is sequential along a line, so the
// parallelism is the number of lines:
//   decompose_x_kernel     one thread per x line, 128 lines per block.  The lines are staged through shared memory in
//                          tiles of 128 lines x 32 samples, loaded and stored by whole warps along x, so global memory is
//                          read and written in 32-sample runs rather than with a stride of W per thread.  It also converts
//                          the input dtype and flags a NaN or +-inf.  The causal sweep writes every tile but the last,
//                          which stays in shared memory for the anticausal sweep.
//   decompose_axis_kernel  one thread per y or z line, consecutive threads on consecutive x: every step is a coalesced
//                          row of float64 in place.
// resample_kernel evaluates one output voxel per thread, consecutive threads along output x.  Per axis it reads the
// continuous index c, returns 0 outside [-0.5, N - 0.5), takes the mask (and the "nearest" image) at floor(c + 0.5), and
// for the B-spline the weights of floor(c) - 1 .. floor(c) + 2 (indices mirrored with period 2N - 2) and the 64 taps from
// the coefficient volume (L1 / L2), summed x innermost, then y, then z, from +0.0.  Every product and sum is rounded to
// float64 on its own (__dmul_rn / __dadd_rn / __dsub_rn: no fused multiply-add), so the results are those of
// lungmask_b200.resample.resample_host bit for bit.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <type_traits>

#include "../../include/lungmask_b200.h"
#include "resample.cuh"

namespace lm {
namespace {

constexpr int kRowsX = 128;    // decompose_x_kernel: x lines (and threads) per block
constexpr int kChunk = 32;     // decompose_x_kernel: samples per line in a shared-memory tile (at least kHorizon)
constexpr int kHorizon = 18;   // ceil(ln 1e-10 / ln |z|): the causal sum of lines longer than this is truncated
constexpr int kThreads = 256;
constexpr double kSixth = 1.0 / 6.0;
static_assert(kChunk >= kHorizon, "the initial causal coefficient must come from the first tile");

template <typename T>
__device__ __forceinline__ double load_f64(const T* __restrict__ p, size_t i) {
  if constexpr (std::is_same<T, __half>::value) return (double)__half2float(p[i]);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return (double)__bfloat162float(p[i]);
  else return (double)p[i];
}

// The first causal coefficient of a line of n >= 2 gain-scaled samples v(0 .. n-1).
template <typename V>
__device__ __forceinline__ double initial_causal(V v, int n, const BsplinePole& p) {
  if (n > kHorizon) {
    double s = v(0), zn = p.z;
    for (int k = 1; k < kHorizon; ++k) {
      s = __dadd_rn(s, __dmul_rn(zn, v(k)));
      zn = __dmul_rn(zn, p.z);
    }
    return s;
  }
  double zn = p.z, z2n = p.z;
  for (int k = 0; k < n - 2; ++k) z2n = __dmul_rn(z2n, p.z);   // z^(n-1)
  double s = __dadd_rn(v(0), __dmul_rn(z2n, v(n - 1)));
  z2n = __dmul_rn(z2n, __dmul_rn(z2n, p.inv_z));
  for (int k = 1; k < n - 1; ++k) {
    s = __dadd_rn(s, __dmul_rn(__dadd_rn(zn, z2n), v(k)));
    zn = __dmul_rn(zn, p.z);
    z2n = __dmul_rn(z2n, p.inv_z);
  }
  return __ddiv_rn(s, __dsub_rn(1.0, __dmul_rn(zn, zn)));
}

template <typename T>
__global__ void __launch_bounds__(kRowsX) decompose_x_kernel(const T* __restrict__ vol, double* __restrict__ out,
                                                             unsigned lines, int n, BsplinePole p, int* flag) {
  __shared__ double tile[kRowsX][kChunk + 1];
  const unsigned line0 = blockIdx.x * kRowsX;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, r = threadIdx.x;
  const bool mine = n > 1 && line0 + r < lines;
  const int chunks = (n + kChunk - 1) / kChunk;
  int bad = 0;
  double prev = 0.0, before = 0.0;   // the causal c[j-1] and c[j-2] of this thread's line
  for (int ch = 0; ch < chunks; ++ch) {   // load, convert and scale; the causal sweep
    const int j0 = ch * kChunk, w = min(kChunk, n - j0);
    for (int row = warp; row < kRowsX; row += kRowsX / 32) {
      if (line0 + row < lines && lane < w) {
        const double v = load_f64(vol, (size_t)(line0 + row) * n + j0 + lane);
        if constexpr (!std::is_integral<T>::value) {
          if (!isfinite(v)) bad = 1;
        }
        tile[row][lane] = n > 1 ? __dmul_rn(v, p.gain) : v;
      }
    }
    __syncthreads();
    if (mine) {
      double* t = tile[r];
      int j = 0;
      if (ch == 0) {
        prev = initial_causal([t](int k) { return t[k]; }, n, p);
        t[0] = prev;
        j = 1;
      }
      for (; j < w; ++j) {
        const double c = __dadd_rn(t[j], __dmul_rn(p.z, prev));
        before = prev;
        prev = c;
        t[j] = c;
      }
      if (ch == chunks - 1) t[w - 1] = __dmul_rn(p.anti, __dadd_rn(__dmul_rn(p.z, before), prev));
    }
    __syncthreads();
    if (ch == chunks - 1) break;   // the last tile stays for the anticausal sweep
    for (int row = warp; row < kRowsX; row += kRowsX / 32)
      if (line0 + row < lines && lane < w) out[(size_t)(line0 + row) * n + j0 + lane] = tile[row][lane];
    __syncthreads();
  }
  double next = 0.0;
  for (int ch = chunks - 1; ch >= 0; --ch) {   // the anticausal sweep
    const int j0 = ch * kChunk, w = min(kChunk, n - j0);
    if (ch < chunks - 1) {
      for (int row = warp; row < kRowsX; row += kRowsX / 32)
        if (line0 + row < lines && lane < w) tile[row][lane] = out[(size_t)(line0 + row) * n + j0 + lane];
      __syncthreads();
    }
    if (mine) {
      double* t = tile[r];
      int j = w - 1;
      if (ch == chunks - 1) next = t[j--];
      for (; j >= 0; --j) {
        next = __dmul_rn(p.z, __dsub_rn(next, t[j]));
        t[j] = next;
      }
    }
    __syncthreads();
    for (int row = warp; row < kRowsX; row += kRowsX / 32)
      if (line0 + row < lines && lane < w) out[(size_t)(line0 + row) * n + j0 + lane] = tile[row][lane];
    __syncthreads();
  }
  if (bad) atomicOr(flag, 1);
}

// One line of n >= 2 samples per thread: line l = o * nx + x starts at c + o * outer + x, its samples `stride` apart.
__global__ void __launch_bounds__(kThreads) decompose_axis_kernel(double* __restrict__ c, unsigned lines, unsigned nx,
                                                                  size_t outer, size_t stride, int n, BsplinePole p) {
  const unsigned l = blockIdx.x * kThreads + threadIdx.x;
  if (l >= lines) return;
  double* a = c + (size_t)(l / nx) * outer + l % nx;
  const double gain = p.gain;
  double prev = initial_causal([a, stride, gain](int k) { return __dmul_rn(a[(size_t)k * stride], gain); }, n, p);
  a[0] = prev;
  double before = 0.0;
  for (int k = 1; k < n; ++k) {
    const double v = __dadd_rn(__dmul_rn(a[(size_t)k * stride], gain), __dmul_rn(p.z, prev));
    before = prev;
    prev = v;
    if (k < n - 1) a[(size_t)k * stride] = v;
  }
  double next = __dmul_rn(p.anti, __dadd_rn(__dmul_rn(p.z, before), prev));
  a[(size_t)(n - 1) * stride] = next;
  for (int k = n - 2; k >= 0; --k) {
    next = __dmul_rn(p.z, __dsub_rn(next, a[(size_t)k * stride]));
    a[(size_t)k * stride] = next;
  }
}

__device__ __forceinline__ bool inside(double c, int n) { return c >= -0.5 && c < (double)n - 0.5; }

__device__ __forceinline__ int nearest(double c, int n) {
  const int i = (int)floor(__dadd_rn(c, 0.5));
  return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
}

__device__ __forceinline__ int mirror(int i, int n) {
  if (n == 1) return 0;
  const int p = 2 * n - 2;
  int k = i % p;
  if (k < 0) k += p;
  return k >= n ? p - k : k;
}

// The indices (mirrored) and weights of the cubic B-spline at continuous index c of an axis of n voxels.
__device__ __forceinline__ void taps(double c, int n, int idx[4], double w[4]) {
  const double f = floor(c);
  const double t = __dsub_rn(c, f);
  const double w3 = __dmul_rn(__dmul_rn(__dmul_rn(kSixth, t), t), t);
  const double w0 = __dsub_rn(__dadd_rn(kSixth, __dmul_rn(__dmul_rn(0.5, t), __dsub_rn(t, 1.0))), w3);
  const double w2 = __dsub_rn(__dadd_rn(t, w0), __dmul_rn(2.0, w3));
  w[0] = w0;
  w[1] = __dsub_rn(__dsub_rn(__dsub_rn(1.0, w0), w2), w3);
  w[2] = w2;
  w[3] = w3;
  const int i0 = (int)f - 1;
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = mirror(i0 + k, n);
}

// The clamp range of an integer output type as float64: its min, and the largest float64 not above its max.
template <typename T> struct IntRange;
template <> struct IntRange<uint8_t> { static constexpr double lo = 0.0, hi = 255.0; };
template <> struct IntRange<int8_t> { static constexpr double lo = -128.0, hi = 127.0; };
template <> struct IntRange<int16_t> { static constexpr double lo = -32768.0, hi = 32767.0; };
template <> struct IntRange<int32_t> { static constexpr double lo = -2147483648.0, hi = 2147483647.0; };
template <> struct IntRange<int64_t> { static constexpr double lo = -9223372036854775808.0, hi = 9223372036854774784.0; };

template <typename T>
__device__ __forceinline__ T cast_out(double v) {
  if constexpr (std::is_same<T, double>::value) {
    return v;
  } else if constexpr (std::is_same<T, float>::value) {
    return __double2float_rn(v);
  } else if constexpr (std::is_same<T, __half>::value) {
    return __double2half(v);
  } else if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    return __float2bfloat16_rn(__double2float_rn(v));
  } else {
    v = v < IntRange<T>::lo ? IntRange<T>::lo : v;
    v = v > IntRange<T>::hi ? IntRange<T>::hi : v;
    return (T)__double2ll_rz(v);
  }
}

template <typename T, int INTERP>
__global__ void __launch_bounds__(kThreads) resample_kernel(const T* __restrict__ vol, const double* __restrict__ coeff,
                                                            const uint8_t* __restrict__ mask, int n0, int n1, int n2,
                                                            const double* __restrict__ cz, const double* __restrict__ cy,
                                                            const double* __restrict__ cx, unsigned m1, unsigned m2,
                                                            unsigned total, T* __restrict__ out,
                                                            uint8_t* __restrict__ out_mask, int* flag) {
  const unsigned i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= total) return;
  const unsigned kx = i % m2, r = i / m2;
  const unsigned ky = r % m1, kz = r / m1;
  const double x = cx[kx], y = cy[ky], z = cz[kz];
  if (!(inside(x, n2) && inside(y, n1) && inside(z, n0))) {
    out[i] = cast_out<T>(0.0);
    out_mask[i] = 0;
    return;
  }
  const size_t near = ((size_t)nearest(z, n0) * n1 + nearest(y, n1)) * n2 + nearest(x, n2);
  out_mask[i] = mask[near];
  double v;
  if constexpr (INTERP == LM_RESAMPLE_NEAREST) {
    v = load_f64(vol, near);
  } else {
    int ix[4], iy[4], iz[4];
    double wx[4], wy[4], wz[4];
    taps(x, n2, ix, wx);
    taps(y, n1, iy, wy);
    taps(z, n0, iz, wz);
    v = 0.0;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      double sy = 0.0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const double* row = coeff + ((size_t)iz[a] * n1 + iy[b]) * n2;
        double sx = 0.0;
#pragma unroll
        for (int c = 0; c < 4; ++c) sx = __dadd_rn(sx, __dmul_rn(wx[c], __ldg(row + ix[c])));
        sy = __dadd_rn(sy, __dmul_rn(wy[b], sx));
      }
      v = __dadd_rn(v, __dmul_rn(wz[a], sy));
    }
  }
  if (!isfinite(v)) atomicOr(flag, 1);
  out[i] = cast_out<T>(v);
}

#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

// Runs f<T>() for the element type of an LM_DTYPE_* code; -1 for an unknown code.
template <typename F>
int by_dtype(int dtype, F&& f) {
  switch (dtype) {
    case LM_DTYPE_U8: return f(uint8_t{});
    case LM_DTYPE_I8: return f(int8_t{});
    case LM_DTYPE_I16: return f(int16_t{});
    case LM_DTYPE_I32: return f(int32_t{});
    case LM_DTYPE_I64: return f(int64_t{});
    case LM_DTYPE_F16: return f(__half{});
    case LM_DTYPE_BF16: return f(__nv_bfloat16{});
    case LM_DTYPE_F32: return f(float{});
    case LM_DTYPE_F64: return f(double{});
    default: return -1;
  }
}

// Reads the flag after the stream has run the kernels: 0 or LM_ERR_NONFINITE.
int finish(ResampleWork& w, cudaStream_t st) {
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? LM_ERR_NONFINITE : 0;
}

}  // namespace

int ResampleWork::reserve() {
  if (!d_flag) {
    const cudaError_t e = cudaMalloc(&d_flag, sizeof(int));
    if (e != cudaSuccess) { d_flag = nullptr; return (int)e; }
  }
  return 0;
}

void ResampleWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

BsplinePole bspline_pole() {
  BsplinePole p;
  p.z = sqrt(3.0) - 2.0;
  p.gain = (1.0 - p.z) * (1.0 - 1.0 / p.z);
  p.inv_z = 1.0 / p.z;
  p.anti = p.z / (p.z * p.z - 1.0);
  return p;
}

int bspline_coefficients(ResampleWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, double* d_coeff,
                         cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  const BsplinePole p = bspline_pole();
  const unsigned xlines = (unsigned)n0 * (unsigned)n1;   // fewer than 2^32 voxels
  const int rc = by_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    decompose_x_kernel<T><<<(xlines + kRowsX - 1) / kRowsX, kRowsX, 0, st>>>(static_cast<const T*>(d_vol), d_coeff,
                                                                             xlines, n2, p, w.d_flag);
    return (int)cudaGetLastError();
  });
  if (rc) return rc;
  ++*launches;
  const size_t plane = (size_t)n1 * n2;
  if (n1 > 1) {   // y lines: (z, x), samples n2 apart
    const unsigned lines = (unsigned)n0 * (unsigned)n2;
    decompose_axis_kernel<<<(lines + kThreads - 1) / kThreads, kThreads, 0, st>>>(d_coeff, lines, (unsigned)n2, plane,
                                                                                  (size_t)n2, n1, p);
    SC(cudaGetLastError());
    ++*launches;
  }
  if (n0 > 1) {   // z lines: (y, x), samples a plane apart
    const unsigned lines = (unsigned)plane;
    decompose_axis_kernel<<<(lines + kThreads - 1) / kThreads, kThreads, 0, st>>>(d_coeff, lines, (unsigned)n2,
                                                                                  (size_t)n2, plane, n0, p);
    SC(cudaGetLastError());
    ++*launches;
  }
  return finish(w, st);
}

int resample_volume(ResampleWork& w, const void* d_vol, int dtype, const double* d_coeff, const uint8_t* d_mask, int n0,
                    int n1, int n2, const double* d_cz, const double* d_cy, const double* d_cx, int m0, int m1, int m2,
                    int interpolator, void* d_out, uint8_t* d_out_mask, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  const unsigned total = (unsigned)m0 * (unsigned)m1 * (unsigned)m2;   // fewer than 2^32 voxels
  const unsigned grid = (total + kThreads - 1) / kThreads;
  const int rc = by_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    const T* v = static_cast<const T*>(d_vol);
    T* o = static_cast<T*>(d_out);
    if (interpolator == LM_RESAMPLE_NEAREST)
      resample_kernel<T, LM_RESAMPLE_NEAREST><<<grid, kThreads, 0, st>>>(v, nullptr, d_mask, n0, n1, n2, d_cz, d_cy, d_cx,
                                                                         (unsigned)m1, (unsigned)m2, total, o, d_out_mask,
                                                                         w.d_flag);
    else if (interpolator == LM_RESAMPLE_BSPLINE)
      resample_kernel<T, LM_RESAMPLE_BSPLINE><<<grid, kThreads, 0, st>>>(v, d_coeff, d_mask, n0, n1, n2, d_cz, d_cy, d_cx,
                                                                         (unsigned)m1, (unsigned)m2, total, o, d_out_mask,
                                                                         w.d_flag);
    else
      return -1;
    return (int)cudaGetLastError();
  });
  if (rc) return rc;
  ++*launches;
  return finish(w, st);
}

}  // namespace lm
