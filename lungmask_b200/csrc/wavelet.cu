// Stationary one-level wavelet decomposition of a volume, one band per call (lm_wavelet_dev, DESIGN §4.12).
//
// PyRadiomics' getWaveletImage with its defaults (pywt.swtn, level 1, axes (2, 1, 0)): three periodic FIR passes, along
// array axis 2 (x), then 1 (y), then 0 (z).  An odd axis of N voxels is wrapped to N' = N + 1 (index N holds index 0);
// a pass gives out[o] = sum_{j = 0..F-1} f[j] in[(o + F/2 - j) mod N'] for o < N, summed from +0.0 with j ascending,
// every product and every sum rounded to float64 (__dmul_rn / __dadd_rn: no fused multiply-add).  The value at a pad
// index of an axis not yet filtered equals the value at index 0, and a pad index of a filtered axis is never read by a
// later pass for an untrimmed output, so every pass reads the input ring through the index map k -> (k mod N' == N ?
// 0 : k mod N').
//
// One fused kernel per band, from the raw input: a block owns a kTY x kTX tile of (y, x) outputs and walks kZ output
// planes.  Per input plane it stages the tile with its F - 1 halo in shared memory as float64, runs the x pass over the
// (kTY + F - 1) rows into shared memory and the y pass into registers; each thread keeps the last F y-pass values of its
// two voxels in a register ring and emits one z-pass output per plane once the ring is full.  No full-volume
// intermediate exists: the only large buffer is the caller's output.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <type_traits>

#include "../../include/lungmask_b200.h"
#include "wavelet.cuh"

namespace lm {
namespace {

constexpr int kTX = 32, kTY = 16, kZ = 32;   // output tile: 32 x-columns (one warp) by 16 y-rows, 32 z-planes per block
constexpr int kThreads = 256;                // thread (ly, lx) owns the outputs (ly, lx) and (ly + 8, lx) of the tile

// PyWavelets' decomposition low-pass filters (dec_lo); dec_hi[k] = (-1)^(k+1) dec_lo[F-1-k].
constexpr double kCoif1[6] = {-0.01565572813546454, -0.0727326195128539, 0.38486484686420286,
                              0.8525720202122554,   0.3378976624578092,  -0.0727326195128539};
constexpr double kHaar[2] = {0.7071067811865476, 0.7071067811865476};

template <int F>
struct Taps {
  double x[F], y[F], z[F];
};

template <typename T>
__device__ __forceinline__ double load_f64(const T* __restrict__ p, size_t i, int* flag) {
  double v;
  if constexpr (std::is_same<T, __half>::value) v = (double)__half2float(p[i]);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) v = (double)__bfloat162float(p[i]);
  else v = (double)p[i];
  if constexpr (!std::is_integral<T>::value) {
    if (!isfinite(v)) atomicOr(flag, 1);
  }
  return v;
}

// The index of the input ring that padded position k reads: k mod N', and index 0 for the pad index N of an odd axis.
// k lies in [-F, 2^31 + kPW) and N' >= F, so k + N' is a non-negative 32-bit unsigned value (a 32-bit remainder).
__device__ __forceinline__ int ring_index(long long k, int n, int np) {
  const unsigned m = (unsigned)(k + np) % (unsigned)np;
  return m == (unsigned)n ? 0 : (int)m;
}

template <typename T, int F>
__global__ void __launch_bounds__(kThreads) wavelet_kernel(const T* __restrict__ vol, double* __restrict__ out, int n0, int n1,
                                                           int n2, int tiles_x, int tiles_y, Taps<F> f, int* flag) {
  constexpr int kHalo = F - 1 - F / 2;              // output o reads inputs o - kHalo .. o + F/2
  constexpr int kPW = kTX + F - 1, kPH = kTY + F - 1;
  __shared__ double s_in[kPH][kPW];                 // the staged input tile of one plane
  __shared__ double s_x[kPH][kTX];                  // its x pass
  __shared__ int s_xs[kPW], s_ys[kPH];              // the ring indices of the tile's columns and rows
  const int tid = threadIdx.x;
  long long b = blockIdx.x;
  const int x0 = (int)(b % tiles_x) * kTX;
  b /= tiles_x;
  const int y0 = (int)(b % tiles_y) * kTY;
  const int z0 = (int)(b / tiles_y) * kZ;
  const int p0 = n0 + (n0 & 1), p1 = n1 + (n1 & 1), p2 = n2 + (n2 & 1);
  for (int i = tid; i < kPW; i += kThreads) s_xs[i] = ring_index((long long)x0 - kHalo + i, n2, p2);
  for (int i = tid; i < kPH; i += kThreads) s_ys[i] = ring_index((long long)y0 - kHalo + i, n1, p1);
  const int lx = tid % kTX, ly = tid / kTX;
  const int ox = x0 + lx, oy0 = y0 + ly, oy1 = y0 + ly + kThreads / kTX;
  double ring0[F], ring1[F];   // y-pass values of planes c - F + 1 .. c at (oy0, ox) and (oy1, ox)
#pragma unroll
  for (int k = 0; k < F; ++k) ring0[k] = ring1[k] = 0.0;
  const int z_end = min(z0 + kZ, n0);
  const int steps = z_end - z0 + F - 1;
  __syncthreads();
  for (int s = 0; s < steps; ++s) {
    // plane c = z0 - kHalo + s of the padded z axis
    const T* plane = vol + (size_t)ring_index((long long)z0 - kHalo + s, n0, p0) * n1 * n2;
    for (int i = tid; i < kPH * kPW; i += kThreads) {
      const int r = i / kPW, c = i - r * kPW;
      s_in[r][c] = load_f64(plane, (size_t)s_ys[r] * n2 + s_xs[c], flag);
    }
    __syncthreads();
    for (int i = tid; i < kPH * kTX; i += kThreads) {
      const int r = i / kTX, c = i - r * kTX;
      double acc = 0.0;
#pragma unroll
      for (int j = 0; j < F; ++j) acc = __dadd_rn(acc, __dmul_rn(f.x[j], s_in[r][c + F - 1 - j]));
      s_x[r][c] = acc;
    }
    __syncthreads();
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int j = 0; j < F; ++j) {
      a0 = __dadd_rn(a0, __dmul_rn(f.y[j], s_x[ly + F - 1 - j][lx]));
      a1 = __dadd_rn(a1, __dmul_rn(f.y[j], s_x[ly + kThreads / kTX + F - 1 - j][lx]));
    }
#pragma unroll
    for (int k = 0; k < F - 1; ++k) {
      ring0[k] = ring0[k + 1];
      ring1[k] = ring1[k + 1];
    }
    ring0[F - 1] = a0;
    ring1[F - 1] = a1;
    if (s >= F - 1 && ox < n2) {
      // output plane o = c - F/2 reads planes o + F/2 - j = c - j: ring[F - 1 - j]
      const size_t o = (size_t)(z0 + s - (F - 1)) * n1;
      double r0 = 0.0, r1 = 0.0;
#pragma unroll
      for (int j = 0; j < F; ++j) {
        r0 = __dadd_rn(r0, __dmul_rn(f.z[j], ring0[F - 1 - j]));
        r1 = __dadd_rn(r1, __dmul_rn(f.z[j], ring1[F - 1 - j]));
      }
      if (oy0 < n1) out[(o + oy0) * n2 + ox] = r0;
      if (oy1 < n1) out[(o + oy1) * n2 + ox] = r1;
    }
  }
}

#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

template <typename T, int F>
int launch(const T* vol, int n0, int n1, int n2, int band, const double* lo, double* out, int* flag, cudaStream_t st) {
  double hi[F];
  for (int k = 0; k < F; ++k) hi[k] = (k % 2 ? 1.0 : -1.0) * lo[F - 1 - k];
  Taps<F> t;
  for (int k = 0; k < F; ++k) {
    t.x[k] = band & 4 ? hi[k] : lo[k];
    t.y[k] = band & 2 ? hi[k] : lo[k];
    t.z[k] = band & 1 ? hi[k] : lo[k];
  }
  const long long tiles_x = (n2 + kTX - 1) / kTX, tiles_y = (n1 + kTY - 1) / kTY, tiles_z = (n0 + kZ - 1) / kZ;
  const long long blocks = tiles_x * tiles_y * tiles_z;
  if (blocks > 0x7fffffffLL) return -1;
  wavelet_kernel<T, F><<<(unsigned)blocks, kThreads, 0, st>>>(vol, out, n0, n1, n2, (int)tiles_x, (int)tiles_y, t, flag);
  return (int)cudaGetLastError();
}

template <typename T>
int band_t(const void* vol, int n0, int n1, int n2, int wavelet, int band, double* out, int* flag, cudaStream_t st) {
  const T* v = static_cast<const T*>(vol);
  if (wavelet == LM_WAVELET_COIF1) return launch<T, 6>(v, n0, n1, n2, band, kCoif1, out, flag, st);
  if (wavelet == LM_WAVELET_HAAR) return launch<T, 2>(v, n0, n1, n2, band, kHaar, out, flag, st);
  return -1;
}

}  // namespace

int wavelet_taps(int wavelet) { return wavelet == LM_WAVELET_COIF1 ? 6 : wavelet == LM_WAVELET_HAAR ? 2 : 0; }

int WaveletWork::reserve() {
  if (d_flag) return 0;
  const cudaError_t e = cudaMalloc(&d_flag, sizeof(int));
  if (e != cudaSuccess) { d_flag = nullptr; return (int)e; }
  return 0;
}

void WaveletWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

int wavelet_band(WaveletWork& w, const void* d_vol, int dtype, int n0, int n1, int n2, int wavelet, int band, double* d_out,
                 cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  int rc;
  switch (dtype) {
    case LM_DTYPE_U8: rc = band_t<uint8_t>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_I8: rc = band_t<int8_t>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_I16: rc = band_t<int16_t>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_I32: rc = band_t<int32_t>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_I64: rc = band_t<int64_t>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_F16: rc = band_t<__half>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_BF16: rc = band_t<__nv_bfloat16>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_F32: rc = band_t<float>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    case LM_DTYPE_F64: rc = band_t<double>(d_vol, n0, n1, n2, wavelet, band, d_out, w.d_flag, st); break;
    default: return -1;
  }
  if (rc) return rc;
  ++*launches;
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? LM_ERR_NONFINITE : 0;
}

}  // namespace lm
