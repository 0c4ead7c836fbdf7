// Voxel-based GLCM feature maps of one row (lm_glcm_maps_dev, DESIGN §4.16).
//
// One thread per voxel (grid-stride) over the uint8 level map of the discretisation region D (0 outside D).  A voxel
// that is not a centre (level 0, or a mask value outside the row) writes init_value to every requested plane.  A centre
// c gathers the levels of its window W(c), the (2r+1)^3 cube clipped at the array border (0 outside the array), into a
// per-thread array; then, per direction d of texture.OFFSETS, it lists the pairs (v, v + d) of the window with both
// levels non-zero as (min, max) keys, accumulating the exact integer sums, the marginal, difference and sum counts on
// the way, insertion-sorts the keys and walks the cells once.  Every float operation is rounded on its own (__dmul_rn,
// __dadd_rn, __ddiv_rn, __dsqrt_rn) in the sequence of lungmask_b200/glcm_maps.py, including its log2 and exp
// routines, so the maps equal its numpy statement bit for bit.  A level above n_levels sets the error flag.
#include <math.h>

#include <algorithm>

#include "glcm_maps.cuh"
#include "map_common.cuh"

namespace lm {
namespace {

constexpr int kThreads = 128;

using maps::cvt_u128;
using maps::insertion_sort;
using maps::offset;
using maps::u128;
typedef __int128 i128;

// Feature bits, in texture.GLCM_FEATURES order (only the ones that gate work are named).
enum : unsigned { kImc1 = 1u << 12, kImc2 = 1u << 13 };

// glcm_maps.py's constants, bit for bit.
constexpr double kEps = 0x1p-52;
constexpr double kSqrt2 = 0x1.6a09e667f3bcdp+0;
constexpr double kLog2e = 0x1.71547652b82fep+0;
constexpr double kLn2Hi = 0x1.62e42fee00000p-1;
constexpr double kLn2Lo = 0x1.a39ef35793c76p-33;
__constant__ double kLogC[10] = {0x1.5555555555555p-1, 0x1.999999999999ap-2, 0x1.2492492492492p-2, 0x1.c71c71c71c71cp-3,
                                 0x1.745d1745d1746p-3, 0x1.3b13b13b13b14p-3, 0x1.1111111111111p-3, 0x1.e1e1e1e1e1e1ep-4,
                                 0x1.af286bca1af28p-4, 0x1.8618618618618p-4};
__constant__ double kExpC[14] = {0x1.6124613a86d09p-33, 0x1.1eed8eff8d898p-29, 0x1.ae64567f544e4p-26,
                                 0x1.27e4fb7789f5cp-22, 0x1.71de3a556c734p-19, 0x1.a01a01a01a01ap-16,
                                 0x1.a01a01a01a01ap-13, 0x1.6c16c16c16c17p-10, 0x1.1111111111111p-7,
                                 0x1.5555555555555p-5,  0x1.5555555555555p-3,  0x1.0000000000000p-1,
                                 0x1.0000000000000p+0,  0x1.0000000000000p+0};

// glcm_maps.log2_fixed: x = 2^e m, m in (sqrt(1/2), sqrt(2)], s = (m - 1) / (m + 1), ln m = 2 s + s z p(z).
__device__ __forceinline__ double log2_fixed(double x) {
  const bool sub = x < 0x1p-1022;
  const long long bits = __double_as_longlong(__dmul_rn(x, sub ? 0x1p54 : 1.0));
  int e = (int)((bits >> 52) & 0x7ff) - 1023 - (sub ? 54 : 0);
  double m = __longlong_as_double((bits & ((1ll << 52) - 1)) | (1023ll << 52));
  if (m > kSqrt2) {
    m = __dmul_rn(m, 0.5);
    ++e;
  }
  const double f = __dsub_rn(m, 1.0);
  const double s = __ddiv_rn(f, __dadd_rn(f, 2.0));
  const double z = __dmul_rn(s, s);
  double p = kLogC[9];
#pragma unroll
  for (int k = 8; k >= 0; --k) p = __dadd_rn(__dmul_rn(p, z), kLogC[k]);
  const double lnm = __dadd_rn(__dadd_rn(s, s), __dmul_rn(__dmul_rn(s, z), p));
  return __dadd_rn((double)e, __dmul_rn(lnm, kLog2e));
}

// glcm_maps.exp_fixed: k = rint(y log2(e)), r = (y - k ln2_hi) - k ln2_lo, the Taylor polynomial of degree 13, times 2^k.
__device__ __forceinline__ double exp_fixed(double y) {
  const double k = rint(__dmul_rn(y, kLog2e));
  const double r = __dsub_rn(__dsub_rn(y, __dmul_rn(k, kLn2Hi)), __dmul_rn(k, kLn2Lo));
  double p = kExpC[0];
#pragma unroll
  for (int i = 1; i < 14; ++i) p = __dadd_rn(__dmul_rn(p, r), kExpC[i]);
  return __dmul_rn(p, __longlong_as_double(((long long)k + 1023) << 52));
}

__device__ __forceinline__ double cvt_i128(i128 v) { return v < 0 ? -cvt_u128((u128)0 - (u128)v) : cvt_u128((u128)v); }

__device__ __forceinline__ double cvt(long long v) { return __ll2double_rn(v); }

template <int R>
__global__ void __launch_bounds__(kThreads) glcm_maps_kernel(const uint8_t* __restrict__ levels, const uint8_t* __restrict__ mask,
                                                             int n0, int n1, int n2, GlcmMapsArgs a, double* __restrict__ out,
                                                             int* flag) {
  constexpr int E = 2 * R + 1, K = E * E * E, P = E * E * (E - 1);
  uint8_t win[K];
  uint16_t key[P];
  uint16_t px[256], pd[256], ps[512];   // per direction: marginal, |i - j| and i + j counts of P; zero between uses
  unsigned present[8];                  // the levels with px > 0
  for (int k = 0; k < 256; ++k) px[k] = pd[k] = 0;
  for (int k = 0; k < 512; ++k) ps[k] = 0;
  const size_t n = (size_t)n0 * n1 * n2;
  const unsigned bits = a.bits;
  const bool need_h1 = bits & kImc1, need_h2 = bits & kImc2;
  const long long g = a.n_levels, g2 = g * g;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int mv = mask[i];
    if (!levels[i] || !(a.row == 256 ? mv != 0 : mv == a.row)) {
      for (unsigned b = bits, j = 0; b; b &= b - 1, ++j) out[(size_t)j * n + i] = a.init_value;
      continue;
    }
    const int x = (int)(i % n2), y = (int)((i / n2) % n1), z = (int)(i / ((size_t)n1 * n2));
    bool bad = false;
    for (int dz = -R; dz <= R; ++dz)
      for (int dy = -R; dy <= R; ++dy)
        for (int dx = -R; dx <= R; ++dx) {
          const int zz = z + dz, yy = y + dy, xx = x + dx;
          int lv = 0;
          if (zz >= 0 && zz < n0 && yy >= 0 && yy < n1 && xx >= 0 && xx < n2) lv = levels[((size_t)zz * n1 + yy) * n2 + xx];
          if (lv > a.n_levels) bad = true;
          win[((dz + R) * E + dy + R) * E + dx + R] = (uint8_t)lv;
        }
    if (bad) {
      atomicOr(flag, 1);
      continue;
    }
    double acc[kGlcmMapsFeatures];
#pragma unroll
    for (int k = 0; k < kGlcmMapsFeatures; ++k) acc[k] = 0.0;
    int nd = 0;
    for (int d = 0; d < 13; ++d) {
      int dz, dy, dx;
      offset(d, dz, dy, dx);
      int np = 0, kmax = 0, smin = 511, smax = 0;
      long long A = 0, Q = 0, B = 0, D1 = 0, D2 = 0, S2 = 0, S3 = 0, S4 = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) present[k] = 0;
      for (int wz = max(0, -dz); wz < min(E, E - dz); ++wz)
        for (int wy = max(0, -dy); wy < min(E, E - dy); ++wy)
          for (int wx = max(0, -dx); wx < min(E, E - dx); ++wx) {
            const int la = win[(wz * E + wy) * E + wx];
            const int lb = win[((wz + dz) * E + wy + dy) * E + wx + dx];
            if (!la || !lb) continue;
            const int lo = min(la, lb), hi = max(la, lb), s = la + lb, df = hi - lo;
            key[np++] = (uint16_t)(lo << 8 | hi);
            const long long s2 = (long long)s * s;
            A += s;
            Q += la * la + lb * lb;
            B += 2 * la * lb;
            D1 += 2 * df;
            D2 += 2 * df * df;
            S2 += 2 * s2;
            S3 += 2 * s2 * s;
            S4 += 2 * s2 * s2;
            ++px[la];
            ++px[lb];
            present[la >> 5] |= 1u << (la & 31);
            present[lb >> 5] |= 1u << (lb & 31);
            pd[df] += 2;
            ps[s] += 2;
            kmax = max(kmax, df);
            smin = min(smin, s);
            smax = max(smax, s);
          }
      if (!np) continue;
      const long long N = 2 * np;
      const double Nd = cvt(N), NN = cvt(N * N);
      const int tb = (int)(N * (N - 1) / 2 - 1);   // T[N][h] = table[tb + h]
      // cells in (i, j) ascending order
      insertion_sort(key, np);
      double je = 0.0, h1 = 0.0;
      long long e2 = 0;
      int mx = 0, start = 0;
      for (int k = 0; k < np; ++k) {
        if (k + 1 < np && key[k + 1] == key[k]) continue;
        const int U = k + 1 - start, lo = key[k] >> 8, hi = key[k] & 255;
        start = k + 1;
        const bool diag = lo == hi;
        const int Pc = diag ? 2 * U : U;
        e2 += diag ? (long long)Pc * Pc : 2ll * Pc * Pc;
        mx = max(mx, Pc);
        const double t = a.table[tb + Pc];
        je = __dadd_rn(je, diag ? t : __dmul_rn(2.0, t));
        if (need_h1) {
          const double w = __ddiv_rn(cvt((long long)px[lo] * px[hi]), NN);
          const double t1 = __dmul_rn(__ddiv_rn(cvt(Pc), Nd), log2_fixed(__dadd_rn(w, kEps)));
          h1 = __dadd_rn(h1, diag ? t1 : __dmul_rn(2.0, t1));
        }
      }
      // levels ascending: HX, and HXY2 over the level pairs i <= j
      double hx = 0.0, h2 = 0.0;
      for (int wi = 0; wi < 8; ++wi)
        for (unsigned bi = present[wi]; bi; bi &= bi - 1) {
          const int li = wi * 32 + __ffs(bi) - 1;
          hx = __dadd_rn(hx, a.table[tb + px[li]]);
          if (need_h2)
            for (int wj = wi; wj < 8; ++wj)
              for (unsigned bj = wj == wi ? present[wj] & (~0u << (li & 31)) : present[wj]; bj; bj &= bj - 1) {
                const int lj = wj * 32 + __ffs(bj) - 1;
                const double w = __ddiv_rn(cvt((long long)px[li] * px[lj]), NN);
                const double t = __dmul_rn(w, log2_fixed(__dadd_rn(w, kEps)));
                h2 = __dadd_rn(h2, lj == li ? t : __dmul_rn(2.0, t));
              }
          px[li] = 0;   // the later levels read only px[lj >= li' > li]
        }
      // differences ascending
      double de = 0.0, idm = 0.0, idmn = 0.0, id = 0.0, idn = 0.0, iv = 0.0;
      for (int k = 0; k <= kmax; ++k) {
        const long long c = pd[k];
        if (!c) continue;
        pd[k] = 0;
        const long long kk = (long long)k * k;
        de = __dadd_rn(de, a.table[tb + c]);
        idm = __dadd_rn(idm, __ddiv_rn(cvt(c), cvt(N * (1 + kk))));
        idmn = __dadd_rn(idmn, __ddiv_rn(cvt(c * g2), cvt(N * (g2 + kk))));
        id = __dadd_rn(id, __ddiv_rn(cvt(c), cvt(N * (1 + k))));
        idn = __dadd_rn(idn, __ddiv_rn(cvt(c * g), cvt(N * (g + k))));
        if (k) iv = __dadd_rn(iv, __ddiv_rn(cvt(c), cvt(N * kk)));
      }
      // sums ascending
      double se = 0.0;
      for (int s = smin; s <= smax; ++s) {
        const int c = ps[s];
        if (!c) continue;
        ps[s] = 0;
        se = __dadd_rn(se, a.table[tb + c]);
      }
      const i128 Ni = N, Ai = A;
      const long long sq = N * Q - A * A;
      const double hxy1 = -h1, hxy2 = -h2;
      double f[kGlcmMapsFeatures];
      f[0] = __ddiv_rn(cvt(B), Nd);                                        // Autocorrelation
      f[1] = __ddiv_rn(cvt(A), Nd);                                        // JointAverage
      f[2] = __ddiv_rn(cvt_i128(Ni * Ni * Ni * S4 - 8 * Ni * Ni * Ai * S3 + 24 * Ni * Ai * Ai * S2 - 48 * Ai * Ai * Ai * Ai),
                       cvt(N * N * N * N));                                // ClusterProminence
      f[3] = __ddiv_rn(cvt_i128(Ni * Ni * S3 - 6 * Ni * Ai * S2 + 16 * Ai * Ai * Ai), cvt(N * N * N));   // ClusterShade
      f[4] = __ddiv_rn(cvt(N * S2 - 4 * A * A), NN);                       // ClusterTendency
      f[5] = __ddiv_rn(cvt(D2), Nd);                                       // Contrast
      f[6] = sq == 0 ? 1.0 : __ddiv_rn(cvt(N * B - A * A), cvt(sq));       // Correlation
      f[7] = __ddiv_rn(cvt(D1), Nd);                                       // DifferenceAverage
      f[8] = de;                                                           // DifferenceEntropy
      f[9] = __ddiv_rn(cvt(N * D2 - D1 * D1), NN);                         // DifferenceVariance
      f[10] = __ddiv_rn(cvt(e2), NN);                                      // JointEnergy
      f[11] = je;                                                          // JointEntropy
      f[12] = hx == 0.0 ? 0.0 : __ddiv_rn(__dsub_rn(je, hxy1), hx);        // Imc1
      f[13] = 0.0;                                                         // Imc2
      if (need_h2 && hxy2 > je) f[13] = __dsqrt_rn(__dsub_rn(1.0, exp_fixed(__dmul_rn(-2.0, __dsub_rn(hxy2, je)))));
      f[14] = idm;
      f[15] = idmn;
      f[16] = id;
      f[17] = idn;
      f[18] = iv;                                                          // InverseVariance
      f[19] = __ddiv_rn(cvt(mx), Nd);                                      // MaximumProbability
      f[20] = se;                                                          // SumEntropy
      f[21] = __ddiv_rn(cvt(sq), NN);                                      // SumSquares
#pragma unroll
      for (int k = 0; k < kGlcmMapsFeatures; ++k) acc[k] = __dadd_rn(acc[k], f[k]);
      ++nd;
    }
    const double ndd = (double)nd;
    int j = 0;
#pragma unroll
    for (int k = 0; k < kGlcmMapsFeatures; ++k)
      if (bits & (1u << k)) out[(size_t)j++ * n + i] = nd ? __ddiv_rn(acc[k], ndd) : nan;
  }
}

#define SC(x)                              \
  do {                                     \
    const cudaError_t e_ = (x);            \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

template <int R>
int launch(const uint8_t* levels, const uint8_t* mask, int n0, int n1, int n2, const GlcmMapsArgs& a, double* out, int* flag,
           int num_sms, cudaStream_t st, int64_t* launches) {
  auto kernel = glcm_maps_kernel<R>;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t n = (size_t)n0 * n1 * n2;
  const size_t need = (n + kThreads - 1) / kThreads;
  const int grid = (int)std::max<size_t>(std::min<size_t>((size_t)per_sm * num_sms * 4, need), 1);
  kernel<<<grid, kThreads, 0, st>>>(levels, mask, n0, n1, n2, a, out, flag);
  SC(cudaGetLastError());
  ++*launches;
  return 0;
}

}  // namespace

int GlcmMapsWork::reserve() {
  if (d_flag) return 0;
  return (int)cudaMalloc(&d_flag, sizeof(int));
}

void GlcmMapsWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

int glcm_maps(GlcmMapsWork& w, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2,
              const GlcmMapsArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  int rc = -1;
  if (a.radius == 1) rc = launch<1>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (a.radius == 2) rc = launch<2>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (a.radius == 3) rc = launch<3>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (rc) return rc;
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? kGlcmMapsRange : 0;
}

}  // namespace lm
