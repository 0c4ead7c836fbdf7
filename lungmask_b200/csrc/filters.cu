// PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient image types, one float64 image per call
// (lm_image_range_dev, lm_image_filter_dev, lm_gradient_dev; DESIGN §4.13).
//
// The elementwise types need m = max|x| over the whole volume: range_kernel reduces min, max and a non-finite flag per
// block (grid-stride, warp shuffles, then shared memory) into per-block partials that the host copies once and folds.
// Every scalar is then formed on the host in float64 and passed in, so that the device does what numpy does with them:
//   square       t = c x; t t                           c = 1 / sqrt(m)
//   squareroot   x > 0: sqrt(x c); x < 0: -sqrt(-x c)    c = m            (anything else, -0.0 included, is kept)
//   logarithm    x > 0: log(x + 1); x < 0: -log(-(x - 1)); then y s     s = m / log(m + 1)
//   exponential  exp(c x)                               c = log(m) / m
// every product, sum and square root rounded to float64 on its own (__dmul_rn / __dadd_rn / __dsqrt_rn: no fused
// multiply-add).  log and exp are CUDA's (within 1 ulp), not numpy's.  For integer volumes the host instead uploads the
// numpy statement evaluated on min..max and filter_kernel<T, kTable> gathers table[x - min], which is numpy's value by
// construction.
//
// gradient_kernel is ITK's GradientMagnitudeImageFilter: per axis g = ((0 + k0 f[-1]) + k1 f[0]) + k2 f[+1] with
// (k0, k1, k2) = (-0.5, 0, 0.5) / s and neighbours clamped to the edge voxel, then sqrt(((0 + gx^2) + gy^2) + gz^2), in
// that order and rounded the same way.  One thread per voxel, consecutive threads along x, so each warp writes 32
// consecutive float64; the six neighbour reads are served by L1 / L2.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <type_traits>

#include "../../include/lungmask_b200.h"
#include "filters.cuh"

namespace lm {
namespace {

constexpr int kThreads = 256;
constexpr int kTable = 4;   // filter_kernel mode after the four LM_FILTER_* codes: the table gather
constexpr int kFlagNonFinite = 1, kFlagTableMiss = 2;

template <typename T>
__device__ __forceinline__ double load_f64(const T* __restrict__ p, size_t i) {
  if constexpr (std::is_same<T, __half>::value) return (double)__half2float(p[i]);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return (double)__bfloat162float(p[i]);
  else return (double)p[i];
}

template <typename T>
__global__ void __launch_bounds__(kThreads) range_kernel(const T* __restrict__ vol, size_t n, double* __restrict__ partial) {
  double lo = INFINITY, hi = -INFINITY;
  int bad = 0;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
    const double v = load_f64(vol, i);
    if constexpr (!std::is_integral<T>::value) {
      if (!isfinite(v)) { bad = 1; continue; }
    }
    lo = fmin(lo, v);
    hi = fmax(hi, v);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
  }
  __shared__ double s_lo[kThreads / 32], s_hi[kThreads / 32];
  __shared__ int s_bad[kThreads / 32];
  const int warp = threadIdx.x / 32;
  if ((threadIdx.x & 31) == 0) {
    s_lo[warp] = lo;
    s_hi[warp] = hi;
    s_bad[warp] = bad;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kThreads / 32; ++k) {
      lo = fmin(lo, s_lo[k]);
      hi = fmax(hi, s_hi[k]);
      bad |= s_bad[k];
    }
    partial[3 * blockIdx.x] = lo;
    partial[3 * blockIdx.x + 1] = hi;
    partial[3 * blockIdx.x + 2] = bad;
  }
}

template <int MODE>
__device__ __forceinline__ double elementwise(double x, double c) {
  if constexpr (MODE == LM_FILTER_SQUARE) {
    const double t = __dmul_rn(c, x);
    return __dmul_rn(t, t);
  } else if constexpr (MODE == LM_FILTER_SQUAREROOT) {
    if (x > 0.0) return __dsqrt_rn(__dmul_rn(x, c));
    if (x < 0.0) return -__dsqrt_rn(__dmul_rn(-x, c));
    return x;
  } else if constexpr (MODE == LM_FILTER_LOGARITHM) {
    double y = x;
    if (x > 0.0) y = log(__dadd_rn(x, 1.0));
    else if (x < 0.0) y = -log(-__dadd_rn(x, -1.0));
    return __dmul_rn(y, c);
  } else {
    return exp(__dmul_rn(c, x));
  }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads) filter_kernel(const T* __restrict__ vol, size_t n, double c,
                                                          const double* __restrict__ table, long long table_min,
                                                          unsigned long long table_len, double* __restrict__ out,
                                                          int* flag) {
  int bad = 0;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
    if constexpr (MODE == kTable) {
      const unsigned long long k = (unsigned long long)((long long)vol[i] - table_min);
      if (k < table_len) {
        out[i] = table[k];
      } else {
        out[i] = 0.0;
        bad |= kFlagTableMiss;
      }
    } else {
      const double x = load_f64(vol, i);
      if constexpr (!std::is_integral<T>::value) {
        if (!isfinite(x)) bad |= kFlagNonFinite;
      }
      out[i] = elementwise<MODE>(x, c);
    }
  }
  if (bad) atomicOr(flag, bad);
}

struct Stencil {
  double k[3][3];   // per axis (x, y, z): (-0.5, 0, 0.5) * (1 / s)
};

template <typename T>
__global__ void __launch_bounds__(kThreads) gradient_kernel(const T* __restrict__ vol, int n0, int n1, int n2, Stencil st,
                                                            double* __restrict__ out, int* flag) {
  const unsigned n = (unsigned)n0 * (unsigned)n1 * (unsigned)n2;   // fewer than 2^32 voxels
  const unsigned plane = (unsigned)n1 * (unsigned)n2;
  int bad = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * kThreads + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * kThreads) {
    const unsigned v = (unsigned)i;
    const unsigned x = v % (unsigned)n2, r = v / (unsigned)n2;
    const unsigned y = r % (unsigned)n1, z = r / (unsigned)n1;
    const double f0 = load_f64(vol, v);
    if constexpr (!std::is_integral<T>::value) {
      if (!isfinite(f0)) bad = kFlagNonFinite;
    }
    // neighbour offsets, clamped to the edge voxel (an axis of one voxel reads f0 on both sides)
    const unsigned dxm = x ? 1u : 0u, dxp = x + 1 < (unsigned)n2 ? 1u : 0u;
    const unsigned dym = y ? (unsigned)n2 : 0u, dyp = y + 1 < (unsigned)n1 ? (unsigned)n2 : 0u;
    const unsigned dzm = z ? plane : 0u, dzp = z + 1 < (unsigned)n0 ? plane : 0u;
    const double fm[3] = {load_f64(vol, v - dxm), load_f64(vol, v - dym), load_f64(vol, v - dzm)};
    const double fp[3] = {load_f64(vol, v + dxp), load_f64(vol, v + dyp), load_f64(vol, v + dzp)};
    double a = 0.0;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      double g = __dadd_rn(0.0, __dmul_rn(st.k[ax][0], fm[ax]));
      g = __dadd_rn(g, __dmul_rn(st.k[ax][1], f0));
      g = __dadd_rn(g, __dmul_rn(st.k[ax][2], fp[ax]));
      a = __dadd_rn(a, __dmul_rn(g, g));
    }
    out[v] = __dsqrt_rn(a);
  }
  if (bad) atomicOr(flag, bad);
}

#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

unsigned grid_for(size_t n, int num_sms, unsigned cap) {
  const size_t want = (n + kThreads - 1) / kThreads;
  const size_t most = (size_t)(num_sms > 0 ? num_sms : 132) * 16;
  size_t g = want < most ? want : most;
  if (g > cap) g = cap;
  return (unsigned)(g ? g : 1);
}

template <typename T>
int filter_t(const void* vol, size_t n, int type, double c, const double* table, int64_t table_min, int64_t table_len,
             double* out, int* flag, unsigned grid, cudaStream_t st) {
  const T* v = static_cast<const T*>(vol);
  const unsigned long long len = (unsigned long long)table_len;
  if (table) {
    if constexpr (std::is_integral<T>::value)
      filter_kernel<T, kTable><<<grid, kThreads, 0, st>>>(v, n, c, table, (long long)table_min, len, out, flag);
    else
      return -1;
  } else {
    switch (type) {
      case LM_FILTER_SQUARE: filter_kernel<T, LM_FILTER_SQUARE><<<grid, kThreads, 0, st>>>(v, n, c, nullptr, 0, 0, out, flag); break;
      case LM_FILTER_SQUAREROOT: filter_kernel<T, LM_FILTER_SQUAREROOT><<<grid, kThreads, 0, st>>>(v, n, c, nullptr, 0, 0, out, flag); break;
      case LM_FILTER_LOGARITHM: filter_kernel<T, LM_FILTER_LOGARITHM><<<grid, kThreads, 0, st>>>(v, n, c, nullptr, 0, 0, out, flag); break;
      case LM_FILTER_EXPONENTIAL: filter_kernel<T, LM_FILTER_EXPONENTIAL><<<grid, kThreads, 0, st>>>(v, n, c, nullptr, 0, 0, out, flag); break;
      default: return -1;
    }
  }
  return (int)cudaGetLastError();
}

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

// Reads the flag after the stream has run the kernel: 0, LM_ERR_NONFINITE or LM_ERR_TABLE_RANGE.
int finish(FilterWork& w, cudaStream_t st) {
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  if (flag & kFlagNonFinite) return LM_ERR_NONFINITE;
  return flag & kFlagTableMiss ? LM_ERR_TABLE_RANGE : 0;
}

}  // namespace

int FilterWork::reserve() {
  if (!d_flag) {
    const cudaError_t e = cudaMalloc(&d_flag, sizeof(int));
    if (e != cudaSuccess) { d_flag = nullptr; return (int)e; }
  }
  if (!d_partial) {
    const cudaError_t e = cudaMalloc(&d_partial, 3 * kFilterRangeBlocks * sizeof(double));
    if (e != cudaSuccess) { d_partial = nullptr; return (int)e; }
  }
  return 0;
}

void FilterWork::release() {
  if (d_flag) cudaFree(d_flag);
  if (d_partial) cudaFree(d_partial);
  d_flag = nullptr;
  d_partial = nullptr;
}

int image_range(FilterWork& w, const void* d_vol, int dtype, size_t n, double out[2], int num_sms, cudaStream_t st,
                int64_t* launches) {
  SC((cudaError_t)w.reserve());
  const unsigned grid = grid_for(n, num_sms, kFilterRangeBlocks);
  const int rc = by_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    range_kernel<T><<<grid, kThreads, 0, st>>>(static_cast<const T*>(d_vol), n, w.d_partial);
    return (int)cudaGetLastError();
  });
  if (rc) return rc;
  ++*launches;
  double part[3 * kFilterRangeBlocks];
  SC(cudaMemcpyAsync(part, w.d_partial, 3 * grid * sizeof(double), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  double lo = INFINITY, hi = -INFINITY;
  bool bad = false;
  for (unsigned b = 0; b < grid; ++b) {
    lo = fmin(lo, part[3 * b]);
    hi = fmax(hi, part[3 * b + 1]);
    bad |= part[3 * b + 2] != 0.0;
  }
  out[0] = lo;
  out[1] = hi;
  return bad ? LM_ERR_NONFINITE : 0;
}

int image_filter(FilterWork& w, const void* d_vol, int dtype, size_t n, int type, double param, const double* d_table,
                 int64_t table_min, int64_t table_len, double* d_out, int num_sms, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  const unsigned grid = grid_for(n, num_sms, 0xffffffffu);
  const int rc = by_dtype(dtype, [&](auto tag) {
    return filter_t<decltype(tag)>(d_vol, n, type, param, d_table, table_min, table_len, d_out, w.d_flag, grid, st);
  });
  if (rc) return rc;
  ++*launches;
  return finish(w, st);
}

int gradient_magnitude(FilterWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, const double inv_xyz[3],
                       double* d_out, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  Stencil s;
  for (int a = 0; a < 3; ++a) {
    s.k[a][0] = -0.5 * inv_xyz[a];
    s.k[a][1] = 0.0 * inv_xyz[a];
    s.k[a][2] = 0.5 * inv_xyz[a];
  }
  const size_t n = (size_t)n0 * n1 * n2;
  const size_t want = (n + kThreads - 1) / kThreads;
  const unsigned grid = (unsigned)(want < 0x7fffffffu ? want : 0x7fffffffu);
  const int rc = by_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    gradient_kernel<T><<<grid, kThreads, 0, st>>>(static_cast<const T*>(d_vol), n0, n1, n2, s, d_out, w.d_flag);
    return (int)cudaGetLastError();
  });
  if (rc) return rc;
  ++*launches;
  return finish(w, st);
}

}  // namespace lm
