// Voxel-based GLSZM, GLRLM, GLDM and NGTDM feature maps of one row (lm_texture_maps_dev, DESIGN §4.17).
//
// One thread per voxel (grid-stride) over the uint8 level map of the discretisation region D (0 outside D), one
// instantiation per (class, radius).  A voxel that is not a centre (level 0, or a mask value outside the row) writes
// init_value to every requested plane.  A centre gathers the levels of its window W(c) once into a per-thread array and
// builds its class's items there: GLSZM a union-find over the window's positions (zones), GLRLM one run walk per
// direction, GLDM and NGTDM 26 neighbour reads per candidate.  The item keys (level << 9 | size) are insertion-sorted and
// walked once by the zone-list evaluator; NGTDM keeps per-level counts and sums instead.  Every float operation is
// rounded on its own (__dmul_rn, __dadd_rn, __ddiv_rn) in the sequence of lungmask_b200/texture_maps.py, so the maps
// equal its numpy statement bit for bit.  A level above n_levels sets the error flag.
#include <algorithm>

#include "map_common.cuh"
#include "texture_maps.cuh"

namespace lm {
namespace {

constexpr int kThreads = 128;
constexpr long long kLcm = 26771144400ll;   // lcm(1..26): L / W is an integer for every neighbour count W

using maps::cvt_u128;
using maps::insertion_sort;
using maps::offset;
using maps::u128;

// The GLSZM feature of each GLDM feature (texture._GLDM_AS_GLSZM).
__constant__ int kGldmOf[14] = {0, 1, 2, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15};

__device__ __forceinline__ double cvt(long long v) { return __ll2double_rn(v); }

// The zone-list evaluator: key[0..n) sorted item keys (level << 9 | size), np the window's candidates; hs a size
// histogram at zero, left at zero.  -> f, the 16 features in texture.GLSZM_FEATURES order.
__device__ __forceinline__ void zone_features(const uint32_t* key, int n, int np, const double* table, uint16_t* hs,
                                              double* f) {
  const long long nz = n;
  const int tb = n * (n - 1) / 2 - 1;   // T[Nz][h] = table[tb + h]
  long long si = 0, si2 = 0, ss = 0, ss2 = 0, sx = 0, gi = 0, gcur = 0;
  int glev = -1, smax = 0, start = 0;
  double a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0, a5 = 0.0, ze = 0.0;
  for (int k = 0; k < n; ++k) {
    if (k + 1 < n && key[k + 1] == key[k]) continue;
    const long long c = k + 1 - start;
    start = k + 1;
    const int i = key[k] >> 9, s = key[k] & 511;
    const long long ii = (long long)i * i, s2 = (long long)s * s;
    si += c * i;
    si2 += c * ii;
    ss += c * s;
    ss2 += c * s2;
    sx += c * ii * s2;
    if (i != glev) {
      gi += gcur * gcur;
      gcur = 0;
      glev = i;
    }
    gcur += c;
    hs[s] += (uint16_t)c;
    smax = max(smax, s);
    const double cf = cvt(c);
    a1 = __dadd_rn(a1, __ddiv_rn(cf, cvt(s2)));
    a2 = __dadd_rn(a2, __ddiv_rn(cf, cvt(ii)));
    a3 = __dadd_rn(a3, __ddiv_rn(cf, cvt(ii * s2)));
    a4 = __dadd_rn(a4, __ddiv_rn(cvt(c * ii), cvt(s2)));
    a5 = __dadd_rn(a5, __ddiv_rn(cvt(c * s2), cvt(ii)));
    ze = __dadd_rn(ze, table[tb + c]);
  }
  gi += gcur * gcur;
  long long gs = 0;
  for (int s = 1; s <= smax; ++s) {
    const long long h = hs[s];
    gs += h * h;
    hs[s] = 0;
  }
  const double N = cvt(nz), NN = cvt(nz * nz);
  f[0] = __ddiv_rn(a1, N);                         // SmallAreaEmphasis
  f[1] = __ddiv_rn(cvt(ss2), N);                   // LargeAreaEmphasis
  f[2] = __ddiv_rn(cvt(gi), N);                    // GrayLevelNonUniformity
  f[3] = __ddiv_rn(cvt(gi), NN);                   // GrayLevelNonUniformityNormalized
  f[4] = __ddiv_rn(cvt(gs), N);                    // SizeZoneNonUniformity
  f[5] = __ddiv_rn(cvt(gs), NN);                   // SizeZoneNonUniformityNormalized
  f[6] = __ddiv_rn(N, cvt(np));                    // ZonePercentage
  f[7] = __ddiv_rn(cvt(nz * si2 - si * si), NN);   // GrayLevelVariance
  f[8] = __ddiv_rn(cvt(nz * ss2 - ss * ss), NN);   // ZoneVariance
  f[9] = ze;                                       // ZoneEntropy
  f[10] = __ddiv_rn(a2, N);                        // LowGrayLevelZoneEmphasis
  f[11] = __ddiv_rn(cvt(si2), N);                  // HighGrayLevelZoneEmphasis
  f[12] = __ddiv_rn(a3, N);                        // SmallAreaLowGrayLevelEmphasis
  f[13] = __ddiv_rn(a4, N);                        // SmallAreaHighGrayLevelEmphasis
  f[14] = __ddiv_rn(a5, N);                        // LargeAreaLowGrayLevelEmphasis
  f[15] = __ddiv_rn(cvt(sx), N);                   // LargeAreaHighGrayLevelEmphasis
}

template <int E>
__device__ __forceinline__ bool inside(int z, int y, int x) {
  return z >= 0 && z < E && y >= 0 && y < E && x >= 0 && x < E;
}

template <int C, int R>
__global__ void __launch_bounds__(kThreads) texture_maps_kernel(const uint8_t* __restrict__ levels,
                                                                const uint8_t* __restrict__ mask, int n0, int n1, int n2,
                                                                TextureMapsArgs a, double* __restrict__ out, int* flag) {
  constexpr int E = 2 * R + 1, K = E * E * E;
  constexpr int NF = texture_maps_features(C);
  constexpr int MAXS = C == kTexMapsGlszm ? K : C == kTexMapsGlrlm ? E : 27;   // the largest item size
  uint8_t win[K];
  const size_t n = (size_t)n0 * n1 * n2;
  const unsigned bits = a.bits;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  uint16_t hs[MAXS + 1];
  for (int s = 0; s <= MAXS; ++s) hs[s] = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int mv = mask[i];
    if (!levels[i] || !(a.row == 256 ? mv != 0 : mv == a.row)) {
      for (unsigned b = bits, j = 0; b; b &= b - 1, ++j) out[(size_t)j * n + i] = a.init_value;
      continue;
    }
    const int x = (int)(i % n2), y = (int)((i / n2) % n1), z = (int)(i / ((size_t)n1 * n2));
    bool bad = false;
    int np = 0;
    for (int dz = -R; dz <= R; ++dz)
      for (int dy = -R; dy <= R; ++dy)
        for (int dx = -R; dx <= R; ++dx) {
          const int zz = z + dz, yy = y + dy, xx = x + dx;
          int lv = 0;
          if (zz >= 0 && zz < n0 && yy >= 0 && yy < n1 && xx >= 0 && xx < n2) lv = levels[((size_t)zz * n1 + yy) * n2 + xx];
          if (lv > a.n_levels) bad = true;
          np += lv != 0;
          win[((dz + R) * E + dy + R) * E + dx + R] = (uint8_t)lv;
        }
    if (bad) {
      atomicOr(flag, 1);
      continue;
    }
    double g[16];
    if constexpr (C == kTexMapsGlszm) {
      // zones: union-find over the window's positions, each root the zone's first position
      int16_t par[K];
      uint32_t key[K];
      for (int p = 0; p < K; ++p) {
        par[p] = (int16_t)p;
        key[p] = 0;
      }
      for (int wz = 0; wz < E; ++wz)
        for (int wy = 0; wy < E; ++wy)
          for (int wx = 0; wx < E; ++wx) {
            const int p = (wz * E + wy) * E + wx, lv = win[p];
            if (!lv) continue;
            for (int d = 0; d < 13; ++d) {
              int dz, dy, dx;
              offset(d, dz, dy, dx);
              if (!inside<E>(wz + dz, wy + dy, wx + dx)) continue;
              const int q = p + (dz * E + dy) * E + dx;
              if (win[q] != lv) continue;
              int ra = p, rb = q;
              while (par[ra] != ra) ra = par[ra] = par[par[ra]];
              while (par[rb] != rb) rb = par[rb] = par[par[rb]];
              if (ra < rb) par[rb] = (int16_t)ra;
              else if (rb < ra) par[ra] = (int16_t)rb;
            }
          }
      // roots are the smallest position of their zone and par[p] <= p, so one ascending pass finds every root
      for (int p = 0; p < K; ++p)
        if (win[p]) {
          par[p] = par[par[p]];
          ++key[par[p]];
        }
      int nk = 0;
      for (int p = 0; p < K; ++p)
        if (win[p] && par[p] == p) {
          const uint32_t size = key[p];
          key[nk++] = (uint32_t)win[p] << 9 | size;   // nk <= p: the slot was read already
        }
      insertion_sort(key, nk);
      zone_features(key, nk, np, a.table, hs, g);
    } else if constexpr (C == kTexMapsGlrlm) {
      uint32_t key[K];
      for (int k = 0; k < 16; ++k) g[k] = 0.0;
      for (int d = 0; d < 13; ++d) {
        int dz, dy, dx;
        offset(d, dz, dy, dx);
        int nk = 0;
        for (int wz = 0; wz < E; ++wz)
          for (int wy = 0; wy < E; ++wy)
            for (int wx = 0; wx < E; ++wx) {
              const int lv = win[(wz * E + wy) * E + wx];
              if (!lv) continue;
              if (inside<E>(wz - dz, wy - dy, wx - dx) && win[((wz - dz) * E + wy - dy) * E + wx - dx] == lv) continue;
              int len = 1;
              for (int t = 1; t < E; ++t) {
                const int qz = wz + t * dz, qy = wy + t * dy, qx = wx + t * dx;
                if (!inside<E>(qz, qy, qx) || win[(qz * E + qy) * E + qx] != lv) break;
                ++len;
              }
              key[nk++] = (uint32_t)lv << 9 | (uint32_t)len;
            }
        insertion_sort(key, nk);
        double f[16];
        zone_features(key, nk, np, a.table, hs, f);
#pragma unroll
        for (int k = 0; k < 16; ++k) g[k] = __dadd_rn(g[k], f[k]);
      }
#pragma unroll
      for (int k = 0; k < 16; ++k) g[k] = __ddiv_rn(g[k], 13.0);
    } else if constexpr (C == kTexMapsGldm) {
      uint32_t key[K];
      int nk = 0;
      for (int wz = 0; wz < E; ++wz)
        for (int wy = 0; wy < E; ++wy)
          for (int wx = 0; wx < E; ++wx) {
            const int lv = win[(wz * E + wy) * E + wx];
            if (!lv) continue;
            int c = 0;
            for (int dz = -1; dz <= 1; ++dz)
              for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                  if (!(dz | dy | dx) || !inside<E>(wz + dz, wy + dy, wx + dx)) continue;
                  const int lq = win[((wz + dz) * E + wy + dy) * E + wx + dx];
                  c += lq && abs(lq - lv) <= a.alpha;
                }
            key[nk++] = (uint32_t)lv << 9 | (uint32_t)(c + 1);
          }
      insertion_sort(key, nk);
      double f[16];
      zone_features(key, nk, np, a.table, hs, f);
#pragma unroll
      for (int k = 0; k < 14; ++k) g[k] = f[kGldmOf[k]];
    } else {
      // NGTDM: per level i the voxels with neighbours (n_i) and sigma_i = sum |W i - S| (L / W), exact
      uint16_t cnt[256];
      long long sig[256];
      unsigned present[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) present[k] = 0;
      for (int wz = 0; wz < E; ++wz)
        for (int wy = 0; wy < E; ++wy)
          for (int wx = 0; wx < E; ++wx) {
            const int lv = win[(wz * E + wy) * E + wx];
            if (!lv) continue;
            int w = 0, s = 0;
            for (int dz = -1; dz <= 1; ++dz)
              for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                  if (!(dz | dy | dx) || !inside<E>(wz + dz, wy + dy, wx + dx)) continue;
                  const int lq = win[((wz + dz) * E + wy + dy) * E + wx + dx];
                  w += lq != 0;
                  s += lq;
                }
            if (!w) continue;
            if (!(present[lv >> 5] & (1u << (lv & 31)))) {
              present[lv >> 5] |= 1u << (lv & 31);
              cnt[lv] = 0;
              sig[lv] = 0;
            }
            ++cnt[lv];
            sig[lv] += (long long)abs(w * lv - s) * (kLcm / w);
          }
      long long nvp = 0, ngp = 0, X = 0, Sg = 0, M1 = 0, M2 = 0, J1 = 0, J2 = 0, B = 0;
      double comp = 0.0;
      for (int wi = 0; wi < 8; ++wi)
        for (unsigned bi = present[wi]; bi; bi &= bi - 1) {
          const long long li = wi * 32 + __ffs(bi) - 1, ni = cnt[li], si = sig[li];
          nvp += ni;
          ++ngp;
          X += ni * si;
          Sg += si;
          M1 += ni * li;
          M2 += ni * li * li;
          J1 += li;
          J2 += li * li;
          for (int wj = wi; wj < 8; ++wj)
            for (unsigned bj = wj == wi ? present[wj] & ~(~0u >> (31 - (int)(li & 31))) : present[wj]; bj; bj &= bj - 1) {
              const long long lj = wj * 32 + __ffs(bj) - 1, nj = cnt[lj];
              B += llabs(li * ni - lj * nj);
              comp = __dadd_rn(comp, __ddiv_rn(cvt_u128((u128)(2 * (lj - li)) * (u128)(ni * si + nj * sig[lj])),
                                               cvt(kLcm * (ni + nj))));
            }
        }
      B *= 2;
      if (!nvp) {
        for (int k = 0; k < 5; ++k) g[k] = nan;
      } else {
        const long long Q = 2 * (nvp * M2 - M1 * M1), Y = 2 * (ngp * M2 - 2 * M1 * J1 + nvp * J2);
        g[0] = X == 0 ? 1e6 : __ddiv_rn(cvt(kLcm * nvp), cvt(X));                                     // Coarseness
        g[1] = ngp > 1 ? __dmul_rn(__ddiv_rn(cvt(Q), cvt(nvp * nvp * ngp * (ngp - 1))), __ddiv_rn(cvt(Sg), cvt(kLcm * nvp)))
                       : 0.0;                                                                         // Contrast
        g[2] = B == 0 ? 0.0 : __ddiv_rn(cvt(X), cvt_u128((u128)kLcm * (u128)B));                     // Busyness
        g[3] = __ddiv_rn(comp, cvt(nvp));                                                            // Complexity
        g[4] = Sg == 0 ? 0.0 : __ddiv_rn(cvt_u128((u128)kLcm * (u128)Y), cvt(nvp * Sg));             // Strength
      }
    }
    int j = 0;
#pragma unroll
    for (int k = 0; k < NF; ++k)
      if (bits & (1u << k)) out[(size_t)j++ * n + i] = g[k];
  }
}

#define SC(x)                              \
  do {                                     \
    const cudaError_t e_ = (x);            \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

template <int C, int R>
int launch(const uint8_t* levels, const uint8_t* mask, int n0, int n1, int n2, const TextureMapsArgs& a, double* out,
           int* flag, int num_sms, cudaStream_t st, int64_t* launches) {
  auto kernel = texture_maps_kernel<C, R>;
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

template <int C>
int launch_class(const uint8_t* levels, const uint8_t* mask, int n0, int n1, int n2, const TextureMapsArgs& a,
                 double* out, int* flag, int num_sms, cudaStream_t st, int64_t* launches) {
  if (a.radius == 1) return launch<C, 1>(levels, mask, n0, n1, n2, a, out, flag, num_sms, st, launches);
  if (a.radius == 2) return launch<C, 2>(levels, mask, n0, n1, n2, a, out, flag, num_sms, st, launches);
  if (a.radius == 3) return launch<C, 3>(levels, mask, n0, n1, n2, a, out, flag, num_sms, st, launches);
  return -1;
}

}  // namespace

int TextureMapsWork::reserve() {
  if (d_flag) return 0;
  return (int)cudaMalloc(&d_flag, sizeof(int));
}

void TextureMapsWork::release() {
  if (d_flag) cudaFree(d_flag);
  d_flag = nullptr;
}

int texture_maps(TextureMapsWork& w, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2,
                 const TextureMapsArgs& a, double* d_out, int num_sms, cudaStream_t st, int64_t* launches) {
  SC((cudaError_t)w.reserve());
  SC(cudaMemsetAsync(w.d_flag, 0, sizeof(int), st));
  int rc = -1;
  if (a.cls == kTexMapsGlszm) rc = launch_class<kTexMapsGlszm>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (a.cls == kTexMapsGlrlm) rc = launch_class<kTexMapsGlrlm>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (a.cls == kTexMapsGldm) rc = launch_class<kTexMapsGldm>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (a.cls == kTexMapsNgtdm) rc = launch_class<kTexMapsNgtdm>(d_levels, d_mask, n0, n1, n2, a, d_out, w.d_flag, num_sms, st, launches);
  if (rc) return rc;
  int flag = 0;
  SC(cudaMemcpyAsync(&flag, w.d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return flag ? kTexMapsRange : 0;
}

}  // namespace lm
