// PyRadiomics' LoG image type: ITK's LaplacianRecursiveGaussianImageFilter with NormalizeAcrossScale
// (lm_laplacian_of_gaussian_dev; DESIGN §4.20).
//
// Each term d = x, y, z is three separable line passes: the order-0 filter along the two other axes (x, y, z order),
// then the order-2 filter along d; the terms are added to d_out from +0.0 in the order x, y, z.  A line pass is ITK's
// RecursiveSeparableImageFilter::FilterDataArray (Deriche's 4th-order recursion, rows in lungmask_b200/laplacian.py):
// a causal sweep y over x with the taps before the line reading x[0], then an anticausal sweep z over x again with the
// taps after the line reading x[L-1], and out = y + z.  Every product and sum is rounded to float64 on its own
// (__dmul_rn / __dadd_rn / __dsub_rn: no fused multiply-add), and the coefficients come from the host, so the result is
// lungmask_b200.laplacian.log_host bit for bit.  The recursion is sequential along a line, so the parallelism is the
// number of lines, one thread each:
//   log_x_kernel     x lines (the contiguous axis), 128 lines per block.  The lines are staged through shared memory in
//                    tiles of 128 lines x 16 samples, loaded and stored along x by half-warps, so global memory is read
//                    and written in 128-byte runs rather than with a stride of W per thread.  The causal sweep runs
//                    forward over the tiles and keeps the last tile of x and y for the anticausal sweep, which runs
//                    backward.
//   log_axis_kernel  y or z lines, consecutive threads on consecutive x: every step is a coalesced row of float64.
// A pass reads its input `src` twice (once per sweep), writes y to `ytmp` and the result to `dst`; ytmp may be dst
// (each element of y is read before its result is written by the same thread), except in the last pass of a term, whose
// dst is the running sum.  The first pass of a term reads the input in its own dtype and flags a NaN or +-inf.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <type_traits>

#include "../../include/lungmask_b200.h"
#include "laplacian.cuh"

namespace lm {
namespace {

constexpr int kRowsX = 128;   // log_x_kernel: x lines (and threads) per block
constexpr int kChunk = 16;    // log_x_kernel: samples per line in a shared-memory tile (one 128-byte run)
constexpr int kThreads = 256;
constexpr int kStore = 0, kFirst = 1, kAdd = 2;   // how a pass writes dst: v, +0.0 + v, dst + v
static_assert(kRowsX % kChunk == 0, "a tile row is loaded by kChunk consecutive threads");

template <typename T>
__device__ __forceinline__ double load_f64(const T* __restrict__ p, size_t i) {
  if constexpr (std::is_same<T, __half>::value) return (double)__half2float(p[i]);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return (double)__bfloat162float(p[i]);
  else return (double)p[i];
}

// ((a0 b0 + a1 b1) + a2 b2) + a3 b3, each product and sum rounded on its own.
__device__ __forceinline__ double e4(double a0, double b0, double a1, double b1, double a2, double b2, double a3,
                                     double b3) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2)), __dmul_rn(a3, b3));
}

// The causal sweep of one line: x[i-1..i-3] and y[i-1..i-4], x[0] before the line; i samples done so far.
struct Causal {
  double x1, x2, x3, y1, y2, y3, y4;
  int i;
};

__device__ __forceinline__ Causal causal_start(double v) { return Causal{v, v, v, v, v, v, v, 0}; }

__device__ __forceinline__ double causal_step(Causal& s, double x, const LogLine& c) {
  const int i = s.i;
  const double y = __dsub_rn(e4(x, c.n[0], s.x1, c.n[1], s.x2, c.n[2], s.x3, c.n[3]),
                             e4(s.y1, i > 0 ? c.d[0] : c.bn[0], s.y2, i > 1 ? c.d[1] : c.bn[1], s.y3,
                                i > 2 ? c.d[2] : c.bn[2], s.y4, i > 3 ? c.d[3] : c.bn[3]));
  s.x3 = s.x2;
  s.x2 = s.x1;
  s.x1 = x;
  s.y4 = s.y3;
  s.y3 = s.y2;
  s.y2 = s.y1;
  s.y1 = y;
  s.i = i + 1;
  return y;
}

// The anticausal sweep of one line: x[j+1..j+4] and z[j+1..j+4], x[L-1] after the line; k samples done so far.
struct Anticausal {
  double x1, x2, x3, x4, z1, z2, z3, z4;
  int k;
};

__device__ __forceinline__ Anticausal anticausal_start(double w) { return Anticausal{w, w, w, w, w, w, w, w, 0}; }

// z[j] from the samples after j, then x[j] joins them.
__device__ __forceinline__ double anticausal_step(Anticausal& s, double x, const LogLine& c) {
  const int k = s.k;
  const double z = __dsub_rn(e4(s.x1, c.m[0], s.x2, c.m[1], s.x3, c.m[2], s.x4, c.m[3]),
                             e4(s.z1, k > 0 ? c.d[0] : c.bm[0], s.z2, k > 1 ? c.d[1] : c.bm[1], s.z3,
                                k > 2 ? c.d[2] : c.bm[2], s.z4, k > 3 ? c.d[3] : c.bm[3]));
  s.x4 = s.x3;
  s.x3 = s.x2;
  s.x2 = s.x1;
  s.x1 = x;
  s.z4 = s.z3;
  s.z3 = s.z2;
  s.z2 = s.z1;
  s.z1 = z;
  s.k = k + 1;
  return z;
}

__device__ __forceinline__ void store(double* dst, size_t g, double v, int mode) {
  if (mode == kAdd) v = __dadd_rn(dst[g], v);
  else if (mode == kFirst) v = __dadd_rn(0.0, v);
  dst[g] = v;
}

template <typename T>
__device__ __forceinline__ void flag_nonfinite(double v, const int* flag, int& bad) {
  if constexpr (!std::is_integral<T>::value) {
    if (flag && !isfinite(v)) bad = 1;
  }
}

// One x line of n samples per thread, line l at src + l * n.  `flag` NULL: the input is not checked.
template <typename T>
__global__ void __launch_bounds__(kRowsX) log_x_kernel(const T* __restrict__ src, double* ytmp, double* dst,
                                                       unsigned lines, int n, LogLine c, int mode, int* flag) {
  __shared__ double xs[kRowsX][kChunk + 1];
  __shared__ double ys[kRowsX][kChunk + 1];
  constexpr int kRowStep = kRowsX / kChunk;
  const unsigned line0 = blockIdx.x * kRowsX;
  const int col = threadIdx.x % kChunk, row0 = threadIdx.x / kChunk, r = threadIdx.x;
  const bool mine = line0 + r < lines;
  const int chunks = (n + kChunk - 1) / kChunk;
  int bad = 0;
  Causal cs;
  for (int ch = 0; ch < chunks; ++ch) {   // load and convert; the causal sweep
    const int j0 = ch * kChunk, w = min(kChunk, n - j0);
    for (int row = row0; row < kRowsX; row += kRowStep) {
      if (line0 + row < lines && col < w) {
        const double v = load_f64(src, (size_t)(line0 + row) * n + j0 + col);
        flag_nonfinite<T>(v, flag, bad);
        xs[row][col] = v;
      }
    }
    __syncthreads();
    if (mine) {
      if (ch == 0) cs = causal_start(xs[r][0]);
      for (int j = 0; j < w; ++j) ys[r][j] = causal_step(cs, xs[r][j], c);
    }
    __syncthreads();
    if (ch == chunks - 1) break;   // the last tile of x and y stays for the anticausal sweep
    for (int row = row0; row < kRowsX; row += kRowStep)
      if (line0 + row < lines && col < w) ytmp[(size_t)(line0 + row) * n + j0 + col] = ys[row][col];
    __syncthreads();
  }
  Anticausal as;
  for (int ch = chunks - 1; ch >= 0; --ch) {   // the anticausal sweep; out = y + z
    const int j0 = ch * kChunk, w = min(kChunk, n - j0);
    if (ch < chunks - 1) {
      for (int row = row0; row < kRowsX; row += kRowStep) {
        if (line0 + row < lines && col < w) {
          const size_t g = (size_t)(line0 + row) * n + j0 + col;
          xs[row][col] = load_f64(src, g);
          ys[row][col] = ytmp[g];
        }
      }
      __syncthreads();
    }
    if (mine) {
      if (ch == chunks - 1) as = anticausal_start(xs[r][w - 1]);
      for (int j = w - 1; j >= 0; --j) ys[r][j] = __dadd_rn(ys[r][j], anticausal_step(as, xs[r][j], c));
    }
    __syncthreads();
    for (int row = row0; row < kRowsX; row += kRowStep)
      if (line0 + row < lines && col < w) store(dst, (size_t)(line0 + row) * n + j0 + col, ys[row][col], mode);
    __syncthreads();
  }
  if (bad) atomicOr(flag, 1);
}

// One line of n samples per thread: line l = o * nx + x starts at o * outer + x, its samples `stride` apart.
template <typename T>
__global__ void __launch_bounds__(kThreads) log_axis_kernel(const T* __restrict__ src, double* ytmp, double* dst,
                                                            unsigned lines, unsigned nx, size_t outer, size_t stride,
                                                            int n, LogLine c, int mode, int* flag) {
  const unsigned l = blockIdx.x * kThreads + threadIdx.x;
  if (l >= lines) return;
  const size_t base = (size_t)(l / nx) * outer + l % nx;
  int bad = 0;
  Causal cs;
  for (int k = 0; k < n; ++k) {
    const size_t g = base + (size_t)k * stride;
    const double x = load_f64(src, g);
    flag_nonfinite<T>(x, flag, bad);
    if (k == 0) cs = causal_start(x);
    ytmp[g] = causal_step(cs, x, c);
  }
  Anticausal as;
  for (int k = n - 1; k >= 0; --k) {
    const size_t g = base + (size_t)k * stride;
    const double x = load_f64(src, g);
    if (k == n - 1) as = anticausal_start(x);
    store(dst, g, __dadd_rn(ytmp[g], anticausal_step(as, x, c)), mode);
  }
  if (bad) atomicOr(flag, 1);
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

// Deriche's constants as ITK's RecursiveGaussianImageFilter states them.
constexpr double kA1[3] = {1.3530, -0.6724, -1.3563}, kB1[3] = {1.8151, -3.4327, 5.2318};
constexpr double kA2[3] = {-0.3531, 0.6724, 0.3446}, kB2[3] = {0.0902, 0.6100, -2.2355};
constexpr double kW1 = 0.6681, kL1 = -1.3932, kW2 = 2.0787, kL2 = -1.3732;

// libm's sin, cos and exp, one per function: the compiler does not merge a sin and a cos of one argument into sincos,
// so each value is the one Python's math module gives for the same argument.
__attribute__((noinline)) double libm_sin(double x) { return sin(x); }
__attribute__((noinline)) double libm_cos(double x) { return cos(x); }
__attribute__((noinline)) double libm_exp(double x) { return exp(x); }

struct Trig {
  double S1, S2, C1, C2, E1, E2;
};

Trig trig(double sd) {
  return Trig{libm_sin(kW1 / sd), libm_sin(kW2 / sd), libm_cos(kW1 / sd), libm_cos(kW2 / sd), libm_exp(kL1 / sd),
              libm_exp(kL2 / sd)};
}

struct Numerator {
  double n[4], sn, dn, en;
};

Numerator numerator(double a1, double b1, double a2, double b2, const Trig& t) {
  const double S1 = t.S1, S2 = t.S2, C1 = t.C1, C2 = t.C2, E1 = t.E1, E2 = t.E2;
  const double N0 = a1 + a2;
  double N1 = E2 * (b2 * S2 - (a2 + 2 * a1) * C2);
  N1 = N1 + E1 * (b1 * S1 - (a1 + 2 * a2) * C1);
  double N2 = (a1 + a2) * C2 * C1;
  N2 = N2 - (b1 * C2 * S1 + b2 * C1 * S2);
  N2 = N2 * (2 * E1 * E2);
  N2 = N2 + (a2 * E1 * E1 + a1 * E2 * E2);
  double N3 = E2 * E1 * E1 * (b2 * S2 - a2 * C2);
  N3 = N3 + E1 * E2 * E2 * (b1 * S1 - a1 * C1);
  return Numerator{{N0, N1, N2, N3}, N0 + N1 + N2 + N3, N1 + 2 * N2 + 3 * N3, N1 + 4 * N2 + 9 * N3};
}

// Reads the flag after the stream has run the kernels: 0 or LM_ERR_NONFINITE.
int finish(LogWork& w, cudaStream_t st) {
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? LM_ERR_NONFINITE : 0;
}

}  // namespace

int LogWork::reserve() {
  if (!d_flag) {
    const cudaError_t e = cudaMalloc(&d_flag, sizeof(int));
    if (e != cudaSuccess) { d_flag = nullptr; return (int)e; }
  }
  return 0;
}

void LogWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

LogLine log_line_coefficients(double sd, int order) {
  const Trig t = trig(sd);
  const double E1 = t.E1, E2 = t.E2, C1 = t.C1, C2 = t.C2;
  const double D1 = -2 * E2 * C2 - 2 * E1 * C1;
  const double D2 = 4 * C2 * C1 * E1 * E2 + E1 * E1 + E2 * E2;
  const double D3 = -2 * C1 * E1 * E2 * E2 - 2 * C2 * E2 * E1 * E1;
  const double D4 = E1 * E1 * E2 * E2;
  const double SD = 1 + D1 + D2 + D3 + D4, DD = D1 + 2 * D2 + 3 * D3 + 4 * D4, ED = D1 + 4 * D2 + 9 * D3 + 16 * D4;
  Numerator N = numerator(kA1[0], kB1[0], kA2[0], kB2[0], t);
  if (order == 0) {
    const double alpha0 = 2 * N.sn / SD - N.n[0];
    for (double& x : N.n) x = x / alpha0;
  } else {
    const Numerator N2 = numerator(kA1[2], kB1[2], kA2[2], kB2[2], t);
    const double beta = -(2 * N2.sn - SD * N2.n[0]) / (2 * N.sn - SD * N.n[0]);
    for (int i = 0; i < 4; ++i) N.n[i] = N2.n[i] + beta * N.n[i];
    const double SN = N2.sn + beta * N.sn, DN = N2.dn + beta * N.dn, EN = N2.en + beta * N.en;
    const double alpha2 = (EN * SD * SD - ED * SN * SD - 2 * DN * DD * SD + 2 * DD * DD * SN) / (SD * SD * SD);
    const double k = sd * sd / alpha2;
    for (double& x : N.n) x = x * k;
  }
  LogLine c;
  const double D[4] = {D1, D2, D3, D4};
  for (int i = 0; i < 4; ++i) {
    c.n[i] = N.n[i];
    c.d[i] = D[i];
  }
  c.m[0] = N.n[1] - D1 * N.n[0];
  c.m[1] = N.n[2] - D2 * N.n[0];
  c.m[2] = N.n[3] - D3 * N.n[0];
  c.m[3] = -D4 * N.n[0];
  const double sum_n = N.n[0] + N.n[1] + N.n[2] + N.n[3];
  const double sum_m = c.m[0] + c.m[1] + c.m[2] + c.m[3];
  for (int i = 0; i < 4; ++i) {
    c.bn[i] = D[i] * sum_n / SD;
    c.bm[i] = D[i] * sum_m / SD;
  }
  return c;
}

int laplacian_of_gaussian(LogWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, const LogLine smooth[3],
                          const LogLine deriv[3], double* d_work0, double* d_work1, double* d_out, cudaStream_t st,
                          int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  const unsigned plane = (unsigned)n1 * (unsigned)n2;   // fewer than 2^32 voxels
  // One pass along axis a (0 = x, 1 = y, 2 = z) of the volume src of element type T.
  auto pass = [&](auto tag, const void* src, int a, const LogLine& c, double* ytmp, double* dst, int mode,
                  int* flag) -> int {
    using T = decltype(tag);
    const T* s = static_cast<const T*>(src);
    if (a == 0) {
      const unsigned lines = (unsigned)n0 * (unsigned)n1;
      log_x_kernel<T><<<(lines + kRowsX - 1) / kRowsX, kRowsX, 0, st>>>(s, ytmp, dst, lines, n2, c, mode, flag);
    } else if (a == 1) {   // y lines: (z, x), samples n2 apart
      const unsigned lines = (unsigned)n0 * (unsigned)n2;
      log_axis_kernel<T><<<(lines + kThreads - 1) / kThreads, kThreads, 0, st>>>(s, ytmp, dst, lines, (unsigned)n2,
                                                                               (size_t)plane, (size_t)n2, n1, c, mode,
                                                                               flag);
    } else {   // z lines: (y, x), samples a plane apart
      log_axis_kernel<T><<<(plane + kThreads - 1) / kThreads, kThreads, 0, st>>>(s, ytmp, dst, plane, (unsigned)n2,
                                                                               (size_t)n2, (size_t)plane, n0, c, mode,
                                                                               flag);
    }
    ++*launches;
    return (int)cudaGetLastError();
  };
  static const int others[3][2] = {{1, 2}, {0, 2}, {0, 1}};
  for (int d = 0; d < 3; ++d) {
    const int a = others[d][0], b = others[d][1];
    int rc = by_dtype(dtype, [&](auto tag) { return pass(tag, d_vol, a, smooth[a], d_work0, d_work0, kStore, w.d_flag); });
    if (rc) return rc;
    rc = pass(double{}, d_work0, b, smooth[b], d_work1, d_work1, kStore, nullptr);
    if (rc) return rc;
    rc = pass(double{}, d_work1, d, deriv[d], d_work0, d_out, d == 0 ? kFirst : kAdd, nullptr);
    if (rc) return rc;
  }
  return finish(w, st);
}

}  // namespace lm
