// Voxel-based first-order feature maps of one row (lm_first_order_maps_dev, DESIGN §4.15).
//
// One thread per voxel (grid-stride).  A voxel outside the ROI (the row's voxels with a non-NaN value) writes
// init_value to every requested plane.  An ROI voxel c gathers the candidates of its window W(c), the (2r+1)^3 cube
// clipped at the array border, in (dz, dy, dx) ascending order, into a per-thread array (local memory), sorts them by
// insertion when an order statistic, the band or the levels are requested, and forms the features in the fixed
// sequence of lungmask_b200/first_order_maps.py, every product, sum, quotient and square root rounded on its own
// (__dmul_rn, __dadd_rn, __ddiv_rn, __dsqrt_rn):
//   exact path  centred int32 d = x - base; S1, S2 in 64 bits and S3, S4 in 128; the moment numerators, the
//               absolute-deviation sums and the energy as integers, each converted to float64 once, correctly rounded
//   float path  float64 values (-0.0 as +0.0); the mean, then the central sums and the energy, then the band's
//               absolute deviations, each a pass over the window in candidate order
// Entropy and Uniformity walk the sorted window's levels in ascending order: one table entry T[n][h] and one (h / n)^2
// per present level.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "../../include/lungmask_b200.h"
#include "first_order_maps.cuh"

namespace lm {
namespace {

constexpr int kThreads = 128;
constexpr int kExactSpan = 1 << 20;

typedef unsigned long long u64;
typedef unsigned __int128 u128;
typedef __int128 i128;

// Feature bits, in first_order.FIRST_ORDER_FEATURES order.
enum : unsigned {
  kP10 = 1u << 0, kP90 = 1u << 1, kEnergy = 1u << 2, kEntropy = 1u << 3, kIqr = 1u << 4, kKurtosis = 1u << 5,
  kMaximum = 1u << 6, kMad = 1u << 7, kMean = 1u << 8, kMedian = 1u << 9, kMinimum = 1u << 10, kRange = 1u << 11,
  kRmad = 1u << 12, kRms = 1u << 13, kSkewness = 1u << 14, kTotalEnergy = 1u << 15, kUniformity = 1u << 16,
  kVariance = 1u << 17
};
constexpr unsigned kNeedSort = kP10 | kP90 | kEntropy | kIqr | kMaximum | kMedian | kMinimum | kRange | kRmad | kUniformity;
constexpr unsigned kNeedMoments = kKurtosis | kSkewness | kVariance;
constexpr unsigned kNeedEnergy = kEnergy | kRms | kTotalEnergy;

template <typename T> constexpr bool kInt = std::is_integral<T>::value;

template <typename T> __device__ __forceinline__ double to_f64(T x) {
  if constexpr (std::is_same<T, __half>::value) return (double)__half2float(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return (double)__bfloat162float(x);
  else if constexpr (kInt<T>) return __ll2double_rn((long long)x);
  else return (double)x;
}

// The correctly rounded float64 of an unsigned 128-bit integer: the top 64 significant bits with every shifted-out bit
// ORed into bit 0 (a sticky bit below the rounding position), rounded to nearest even, scaled by 2^s exactly.
__device__ __forceinline__ double cvt_u128(u128 m) {
  const u64 hi = (u64)(m >> 64), lo = (u64)m;
  if (!hi) return __ull2double_rn(lo);
  const int s = 64 - __clzll((long long)hi);   // 1..64
  u64 top = (u64)(m >> s);
  const u64 out = s == 64 ? lo : (lo & ((1ull << s) - 1));
  if (out) top |= 1ull;
  return __dmul_rn(__ull2double_rn(top), __longlong_as_double((long long)(1023 + s) << 52));
}
__device__ __forceinline__ double cvt_i128(i128 v) {
  return v < 0 ? -cvt_u128((u128)0 - (u128)v) : cvt_u128((u128)v);
}

// numpy's _lerp of percentile(..., method="linear"), each product and sum rounded on its own (stats.cu's np_lerp).
__device__ __forceinline__ double np_lerp(double a, double b, double t) {
  const double diff = __dsub_rn(b, a);
  double r = __dadd_rn(a, __dmul_rn(diff, t));
  if (t >= 0.5) r = __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, t)));
  return r;
}

template <typename T>
__device__ __forceinline__ bool in_roi(const T* vol, const uint8_t* mask, size_t j, int row) {
  const int m = mask[j];
  if (!(row == 256 ? m != 0 : m == row)) return false;
  if constexpr (!kInt<T>) return !isnan(to_f64(vol[j]));
  return true;
}

template <typename T>
__device__ __forceinline__ bool candidate(const T* vol, const uint8_t* mask, size_t j, int row, int masked) {
  if (masked) return in_roi(vol, mask, j, row);
  if constexpr (!kInt<T>) return !isnan(to_f64(vol[j]));
  return true;
}

template <int R> struct Window {
  static constexpr int K = (2 * R + 1) * (2 * R + 1) * (2 * R + 1);
};

// Calls f(j) for every candidate voxel index j of the window of (z, y, x), in (dz, dy, dx) ascending order.
template <int R, typename T, typename F>
__device__ __forceinline__ void for_window(const T* vol, const uint8_t* mask, int n0, int n1, int n2, int z, int y, int x,
                                           int row, int masked, F f) {
  for (int dz = -R; dz <= R; ++dz) {
    const int zz = z + dz;
    if (zz < 0 || zz >= n0) continue;
    for (int dy = -R; dy <= R; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= n1) continue;
      const size_t line = ((size_t)zz * n1 + yy) * n2;
      for (int dx = -R; dx <= R; ++dx) {
        const int xx = x + dx;
        if (xx < 0 || xx >= n2) continue;
        const size_t j = line + xx;
        if (candidate(vol, mask, j, row, masked)) f(j);
      }
    }
  }
}

template <typename K> __device__ __forceinline__ void insertion_sort(K* v, int n) {
  for (int i = 1; i < n; ++i) {
    const K k = v[i];
    int j = i - 1;
    while (j >= 0 && v[j] > k) {
      v[j + 1] = v[j];
      --j;
    }
    v[j + 1] = k;
  }
}

__device__ __forceinline__ void put(double* out, size_t n, size_t i, unsigned bits, unsigned bit, double v) {
  if (bits & bit) out[(size_t)__popc(bits & (bit - 1)) * n + i] = v;
}

// The order statistics of the sorted window xs(k) (k = 0..n-1): P10, P25, P50, P75, P90 by numpy's linear method.
template <typename X> __device__ __forceinline__ void percentiles(X xs, int n, double p[5]) {
  const double q[5] = {0.1, 0.25, 0.5, 0.75, 0.9};
  const double last = (double)(n - 1);
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const double h = __dmul_rn(last, q[k]);
    const double fh = floor(h);
    const bool top = h >= last;
    const int i = top ? n - 1 : (int)fh;
    const int i1 = top ? n - 1 : i + 1;
    const double t = top ? __dadd_rn(h, 1.0) : __dsub_rn(h, fh);
    p[k] = np_lerp(xs(i), xs(i1), t);
  }
}

// Entropy and Uniformity of the sorted window: level(k) non-decreasing in k.
template <typename L>
__device__ __forceinline__ void level_sums(L level, int n, const double* table, double& ent, double& uni) {
  ent = 0.0;
  uni = 0.0;
  const double nd = (double)n;
  const int tb = n * (n - 1) / 2 - 1;
  int start = 0;
  long long prev = level(0);
  for (int k = 1; k <= n; ++k) {
    const long long lv = k < n ? level(k) : -1;
    if (k == n || lv != prev) {
      const int h = k - start;
      ent = __dadd_rn(ent, table[tb + h]);
      const double p = __ddiv_rn((double)h, nd);
      uni = __dadd_rn(uni, __dmul_rn(p, p));
      start = k;
      prev = lv;
    }
  }
}

template <typename T, int R, bool kExact>
__global__ void __launch_bounds__(kThreads) first_order_maps_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask,
                                                                    int n0, int n1, int n2, FomArgs a, double* __restrict__ out,
                                                                    int* flag) {
  constexpr int K = Window<R>::K;
  typedef typename std::conditional<kExact, int, double>::type Key;
  Key key[K];
  const size_t n = (size_t)n0 * n1 * n2;
  const unsigned bits = a.bits;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (!in_roi(vol, mask, i, a.row)) {
      for (unsigned b = bits; b; b &= b - 1) put(out, n, i, bits, b & (0u - b), a.init_value);
      continue;
    }
    const int x = (int)(i % n2), y = (int)((i / n2) % n1), z = (int)(i / ((size_t)n1 * n2));
    int cnt = 0;
    double mean, var = 0.0, skew = 0.0, kurt = 0.0, mad = 0.0, rmad = nan, energy = 0.0;
    double p[5] = {0.0, 0.0, 0.0, 0.0, 0.0}, vmin = 0.0, vmax = 0.0, ent = 0.0, uni = 0.0;
    if constexpr (kExact) {
      u64 s1 = 0, s2 = 0;
      u128 s3 = 0, s4 = 0;
      bool bad = false;
      for_window<R>(vol, mask, n0, n1, n2, z, y, x, a.row, a.masked, [&](size_t j) {
        const u64 d = (u64)((long long)vol[j] - a.base);   // modular: a value below base wraps above the span
        if (d >= (u64)kExactSpan) { bad = true; return; }
        key[cnt++] = (int)d;
        const u64 d2 = d * d;
        s1 += d;
        s2 += d2;
        s3 += (u128)(d2 * d);
        s4 += (u128)d2 * d2;
      });
      if (bad) { atomicOr(flag, 2); continue; }
      const long long nn = cnt;
      const double nd = (double)cnt;
      mean = __ddiv_rn(__ll2double_rn(a.base * nn + (long long)s1), nd);
      if (bits & (kNeedSort | kEntropy | kUniformity)) {
        insertion_sort(key, cnt);
        auto xs = [&](int k) { return __ll2double_rn(a.base + key[k]); };
        percentiles(xs, cnt, p);
        vmin = xs(0);
        vmax = xs(cnt - 1);
        if (bits & (kEntropy | kUniformity)) {
          bool range = false;
          auto level = [&](int k) {
            const long long lv = (a.base + key[k] - a.low) / a.bin_width + 1;
            if (lv < 1 || lv > a.n_levels) range = true;
            return lv;
          };
          level_sums(level, cnt, a.table, ent, uni);
          if (range) { atomicOr(flag, 2); continue; }
        }
        if (bits & kRmad) {
          long long nb = 0, sb = 0;
          for (int k = 0; k < cnt; ++k) {
            const double xv = xs(k);
            if (xv >= p[0] && xv <= p[4]) { ++nb; sb += key[k]; }
          }
          if (nb) {
            long long ab = 0;
            for (int k = 0; k < cnt; ++k) {
              const double xv = xs(k);
              if (xv >= p[0] && xv <= p[4]) { const long long t = nb * key[k] - sb; ab += t < 0 ? -t : t; }
            }
            rmad = __ddiv_rn(__ll2double_rn(ab), (double)(nb * nb));
          }
        }
      }
      if (bits & kMad) {
        long long A = 0;
        for (int k = 0; k < cnt; ++k) { const long long t = nn * key[k] - (long long)s1; A += t < 0 ? -t : t; }
        mad = __ddiv_rn(__ll2double_rn(A), (double)(nn * nn));
      }
      if (bits & kNeedMoments) {
        const long long m2n = nn * (long long)s2 - (long long)(s1 * s1);
        var = __ddiv_rn(__ll2double_rn(m2n), (double)(nn * nn));
        if (m2n != 0) {
          const u128 S1 = s1, S2 = s2, N = (u128)nn;
          const u128 m3n = N * N * s3 - 3 * N * S1 * S2 + 2 * S1 * S1 * S1;
          const u128 m4n = N * N * N * s4 - 4 * N * N * S1 * s3 + 6 * N * S1 * S1 * S2 - 3 * S1 * S1 * S1 * S1;
          skew = __ddiv_rn(__ddiv_rn(cvt_i128((i128)m3n), (double)(nn * nn * nn)), __dmul_rn(var, __dsqrt_rn(var)));
          kurt = __ddiv_rn(cvt_i128((i128)m4n), cvt_u128((u128)m2n * (u128)m2n));
        }
      }
      if (bits & kNeedEnergy) {
        const i128 c = (i128)(a.base + a.shift);
        energy = cvt_i128((i128)s2 + 2 * c * (i128)s1 + (i128)nn * c * c);
      }
    } else {
      double s = 0.0;
      bool inf = false;
      for_window<R>(vol, mask, n0, n1, n2, z, y, x, a.row, a.masked, [&](size_t j) {
        const double v = __dadd_rn(to_f64(vol[j]), 0.0);   // -0.0 as +0.0
        if (isinf(v)) inf = true;
        key[cnt++] = v;
        s = __dadd_rn(s, v);
      });
      if (inf) { atomicOr(flag, 1); continue; }
      const double nd = (double)cnt;
      mean = __ddiv_rn(s, nd);
      if (bits & (kNeedSort | kEntropy | kUniformity)) {
        // the moments below re-read the window in candidate order; the sort only serves the order statistics
        insertion_sort(key, cnt);
        auto xs = [&](int k) { return key[k]; };
        percentiles(xs, cnt, p);
        vmin = key[0];
        vmax = key[cnt - 1];
        if (bits & (kEntropy | kUniformity)) {
          bool range = false;
          auto level = [&](int k) {
            const double f = floor(key[k]);
            long long lv = -1;
            if (f > -9.0e18 && f < 9.0e18) lv = ((long long)f - a.low) / a.bin_width + 1;
            if (lv < 1 || lv > a.n_levels) range = true;
            return lv;
          };
          level_sums(level, cnt, a.table, ent, uni);
          if (range) { atomicOr(flag, 2); continue; }
        }
      }
      const double c = __ll2double_rn(a.shift);
      double m2 = 0.0, m3 = 0.0, m4 = 0.0, ad = 0.0, sb = 0.0;
      int nb = 0;
      const bool band = bits & kRmad;
      if (bits & (kNeedMoments | kMad | kNeedEnergy | kRmad)) {
        for_window<R>(vol, mask, n0, n1, n2, z, y, x, a.row, a.masked, [&](size_t j) {
          const double v = __dadd_rn(to_f64(vol[j]), 0.0);
          const double e = __dsub_rn(v, mean), e2 = __dmul_rn(e, e);
          m2 = __dadd_rn(m2, e2);
          m3 = __dadd_rn(m3, __dmul_rn(e2, e));
          m4 = __dadd_rn(m4, __dmul_rn(e2, e2));
          ad = __dadd_rn(ad, fabs(e));
          const double t = __dadd_rn(v, c);
          energy = __dadd_rn(energy, __dmul_rn(t, t));
          if (band && v >= p[0] && v <= p[4]) { sb = __dadd_rn(sb, v); ++nb; }
        });
      }
      var = __ddiv_rn(m2, nd);
      if (m2 != 0.0) {
        skew = __ddiv_rn(__ddiv_rn(m3, nd), __dmul_rn(var, __dsqrt_rn(var)));
        kurt = __ddiv_rn(__ddiv_rn(m4, nd), __dmul_rn(var, var));
      }
      mad = __ddiv_rn(ad, nd);
      if (band && nb) {
        const double mb = __ddiv_rn(sb, (double)nb);
        double adb = 0.0;
        for_window<R>(vol, mask, n0, n1, n2, z, y, x, a.row, a.masked, [&](size_t j) {
          const double v = __dadd_rn(to_f64(vol[j]), 0.0);
          if (v >= p[0] && v <= p[4]) adb = __dadd_rn(adb, fabs(__dsub_rn(v, mb)));
        });
        rmad = __ddiv_rn(adb, (double)nb);
      }
    }
    const double nd = (double)cnt;
    put(out, n, i, bits, kP10, p[0]);
    put(out, n, i, bits, kP90, p[4]);
    put(out, n, i, bits, kEnergy, energy);
    put(out, n, i, bits, kEntropy, ent);
    put(out, n, i, bits, kIqr, __dsub_rn(p[3], p[1]));
    put(out, n, i, bits, kKurtosis, kurt);
    put(out, n, i, bits, kMaximum, vmax);
    put(out, n, i, bits, kMad, mad);
    put(out, n, i, bits, kMean, mean);
    put(out, n, i, bits, kMedian, p[2]);
    put(out, n, i, bits, kMinimum, vmin);
    put(out, n, i, bits, kRange, __dsub_rn(vmax, vmin));
    put(out, n, i, bits, kRmad, rmad);
    put(out, n, i, bits, kRms, __dsqrt_rn(__ddiv_rn(energy, nd)));
    put(out, n, i, bits, kSkewness, skew);
    put(out, n, i, bits, kTotalEnergy, __dmul_rn(a.voxel_volume, energy));
    put(out, n, i, bits, kUniformity, uni);
    put(out, n, i, bits, kVariance, var);
  }
}

#define SC(x)                              \
  do {                                     \
    const cudaError_t e_ = (x);            \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

template <typename T, int R, bool kExact>
int launch(const T* vol, const uint8_t* mask, int n0, int n1, int n2, const FomArgs& a, double* out, int* flag, int num_sms,
           cudaStream_t st, int64_t* launches) {
  auto kernel = first_order_maps_kernel<T, R, kExact>;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t n = (size_t)n0 * n1 * n2;
  const size_t need = (n + kThreads - 1) / kThreads;
  const int grid = (int)std::max<size_t>(std::min<size_t>((size_t)per_sm * num_sms * 4, need), 1);
  kernel<<<grid, kThreads, 0, st>>>(vol, mask, n0, n1, n2, a, out, flag);
  SC(cudaGetLastError());
  ++*launches;
  return 0;
}

template <typename T>
int run(FomWork& w, const T* vol, const uint8_t* mask, int n0, int n1, int n2, const FomArgs& a, double* out, int num_sms,
        cudaStream_t st, int64_t* launches) {
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  int rc = -1;
  if constexpr (kInt<T>) {
    if (a.exact) {
      if (a.radius == 1) rc = launch<T, 1, true>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
      if (a.radius == 2) rc = launch<T, 2, true>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
      if (a.radius == 3) rc = launch<T, 3, true>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
    }
  }
  if (!a.exact) {
    if (a.radius == 1) rc = launch<T, 1, false>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
    if (a.radius == 2) rc = launch<T, 2, false>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
    if (a.radius == 3) rc = launch<T, 3, false>(vol, mask, n0, n1, n2, a, out, w.d_flag, num_sms, st, launches);
  }
  if (rc) return rc;
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  if (flag & 1) return LM_ERR_NONFINITE;
  if (flag & 2) return kFomRange;
  return 0;
}

}  // namespace

int FomWork::reserve() {
  if (d_flag) return 0;
  return (int)cudaMalloc(&d_flag, sizeof(int));
}

void FomWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

int first_order_maps(FomWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                     const FomArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
#define LM_FOM_CASE(code, T) \
  case code: return run<T>(w, static_cast<const T*>(d_vol), d_mask, n0, n1, n2, a, d_out, num_sms, st, launches)
  switch (dtype) {
    LM_FOM_CASE(LM_DTYPE_U8, uint8_t);
    LM_FOM_CASE(LM_DTYPE_I8, int8_t);
    LM_FOM_CASE(LM_DTYPE_I16, int16_t);
    LM_FOM_CASE(LM_DTYPE_I32, int32_t);
    LM_FOM_CASE(LM_DTYPE_I64, int64_t);
    LM_FOM_CASE(LM_DTYPE_F16, __half);
    LM_FOM_CASE(LM_DTYPE_BF16, __nv_bfloat16);
    LM_FOM_CASE(LM_DTYPE_F32, float);
    LM_FOM_CASE(LM_DTYPE_F64, double);
    default: return -1;
  }
#undef LM_FOM_CASE
}

}  // namespace lm
