// Pre-processing on device: utils.preprocess (utils.py:32-52) = per slice simple_bodymask (utils.py:55-82),
// crop to the body bounding box (utils.py:98-107) and bilinear resize to 256x256 (utils.py:108-110),
// bit-exact with the scipy.ndimage / skimage semantics the reference inherits (oracle/restate.py spells
// them out; every float64 operation below uses explicit round-to-nearest intrinsics so the compiler cannot
// contract a multiply-add and change a rounding).
//
// bodymask_kernel: ONE CTA PER SLICE, everything on a 128x128 thumbnail held as a 128x(4x32)-bit mask in
// shared memory: threshold, closing, hole fill, 2x erosion, largest 4-connected component (union-find in
// shared memory), 2x dilation, and finally the bounding box of component #1 of the 8-connected labelling of
// the nearest-neighbour up-scaled mask - computed on the thumbnail through the monotone index maps, so the
// full-resolution mask is never materialised (it is written only when a caller asks for it).
// resize_kernel: one thread per output pixel, float64 coordinates and accumulation order as scipy's zoom.
#include <atomic>
#include <type_traits>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "../../include/lungmask_b200.h"
#include "preproc.cuh"

namespace lm {
namespace {

constexpr int T = 128;           // thumbnail edge (utils.py:68)
constexpr int WORDS = T / 32;    // 4 words per row
constexpr int NTHREADS = 512;    // one thread per mask word
constexpr uint32_t NONE = 0xFFFFFFFFu;

struct AxisMap {
  double step;  // (n_in-1)/(n_out-1), float64 division exactly as scipy computes it
  int n_in, n_out;
};
__device__ __forceinline__ AxisMap make_axis(int n_in, int n_out) {
  AxisMap a;
  a.n_in = n_in; a.n_out = n_out;
  a.step = n_out > 1 ? __ddiv_rn((double)(n_in - 1), (double)(n_out - 1)) : 0.0;
  return a;
}
// nearest-neighbour source index for output o, or -1 when the coordinate falls outside (mode='constant')
__device__ __forceinline__ int nn_index(const AxisMap& a, int o) {
  if (a.n_out <= 1) return 0;
  const double c = __dmul_rn((double)o, a.step);
  if (c > (double)(a.n_in - 1)) return -1;
  int i = (int)floor(__dadd_rn(c, 0.5));
  return i < 0 ? 0 : (i > a.n_in - 1 ? a.n_in - 1 : i);
}

struct Smem {
  uint32_t bits[2][T][WORDS];
  uint32_t parent[T * T];
  uint32_t area2[T * T / 2];            // component areas as packed 16-bit counters (an area is at most 128 * 128 = 2^14):
                                        // 103 KB instead of 135 KB per CTA, so two slices share an SM
  int first_o[2][T], last_o[2][T];      // [axis][thumb index] -> first / last valid output index mapping to it
  int16_t prevp[2][T], nextp[2][T];     // previous / next PRESENT thumb index along each axis
  uint32_t best_key;
  uint32_t min_root;
  int bb[4];
  int flag;
};

__device__ __forceinline__ uint32_t get_word(const uint32_t (*b)[WORDS], int r, int k) {
  return (r < 0 || r >= T || k < 0 || k >= WORDS) ? 0u : b[r][k];
}
__device__ __forceinline__ uint32_t left_of(const uint32_t (*b)[WORDS], int r, int k) {  // value of neighbour j-1
  return (b[r][k] << 1) | (k > 0 ? (b[r][k - 1] >> 31) : 0u);
}
__device__ __forceinline__ uint32_t right_of(const uint32_t (*b)[WORDS], int r, int k) {  // neighbour j+1
  return (b[r][k] >> 1) | (k < WORDS - 1 ? (b[r][k + 1] << 31) : 0u);
}
// scipy binary_dilation / binary_erosion with the default cross structure and border_value=0
__device__ __forceinline__ uint32_t dilate_cross(const uint32_t (*b)[WORDS], int r, int k) {
  return b[r][k] | left_of(b, r, k) | right_of(b, r, k) | get_word(b, r - 1, k) | get_word(b, r + 1, k);
}
__device__ __forceinline__ uint32_t erode_cross(const uint32_t (*b)[WORDS], int r, int k) {
  return b[r][k] & left_of(b, r, k) & right_of(b, r, k) & get_word(b, r - 1, k) & get_word(b, r + 1, k);
}
__device__ __forceinline__ uint32_t hdil3(const uint32_t (*b)[WORDS], int r, int k) {
  return (r < 0 || r >= T) ? 0u : (b[r][k] | left_of(b, r, k) | right_of(b, r, k));
}

__device__ __forceinline__ uint32_t uf_find(uint32_t* parent, uint32_t i) {
  uint32_t p = parent[i];
  while (p != i) { i = p; p = parent[i]; }
  return i;
}
__device__ __forceinline__ void uf_union(uint32_t* parent, uint32_t a, uint32_t b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { uint32_t t = a; a = b; b = t; }
    const uint32_t old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}
__device__ __forceinline__ bool bit_at(const uint32_t (*b)[WORDS], int r, int c) {
  return (b[r][c >> 5] >> (c & 31)) & 1u;
}

template <typename VT>
__global__ void __launch_bounds__(NTHREADS, 2)   // 64 registers: two CTAs (slices) per SM hide each other's barrier latencies
bodymask_kernel(const VT* __restrict__ vol, int S, int H, int W, int32_t* __restrict__ boxes,
                uint8_t* __restrict__ mask_out) {
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wr = tid / WORDS, wk = tid % WORDS;  // this thread's mask word: row wr, word wk

  for (int s = blockIdx.x; s < S; s += gridDim.x) {
    const VT* img = vol + (size_t)s * H * W;
    const AxisMap dn_y = make_axis(H, T), dn_x = make_axis(W, T);  // zoom(img, 128/shape, order=0), utils.py:68
    const AxisMap up_y = make_axis(T, H), up_x = make_axis(T, W);  // zoom(mask, shape/128, order=0), utils.py:81-82

    // (1) thumbnail + threshold (> -500 HU, utils.py:58,69). Outside samples are cval = 0 (> -500 -> set).
    for (int w = warp; w < T * WORDS; w += NTHREADS / 32) {
      const int r = w / WORDS, k = w % WORDS, c = k * 32 + lane;
      const int iy = nn_index(dn_y, r), ix = nn_index(dn_x, c);
      // (int16 HU, or float HU for float volumes - the reference thresholds whatever dtype it is given)
      const double v = (iy >= 0 && ix >= 0) ? (double)img[(size_t)iy * W + ix] : 0.0;
      const uint32_t word = __ballot_sync(0xffffffffu, v > -500.0);
      if (lane == 0) sm.bits[0][r][k] = word;
    }
    __syncthreads();
    // (2) binary_closing (utils.py:70): dilation then erosion, cross, zero border
    sm.bits[1][wr][wk] = dilate_cross(sm.bits[0], wr, wk);
    __syncthreads();
    sm.bits[0][wr][wk] = erode_cross(sm.bits[1], wr, wk);
    __syncthreads();
    // (3) binary_fill_holes(structure=ones(3,3)) (utils.py:71): background 8-connected to the frame
    {
      const uint32_t bg = ~sm.bits[0][wr][wk];
      uint32_t seed = 0;
      if (wr == 0 || wr == T - 1) seed = 0xFFFFFFFFu;
      if (wk == 0) seed |= 1u;
      if (wk == WORDS - 1) seed |= 0x80000000u;
      uint32_t reach = bg & seed;
      sm.bits[1][wr][wk] = reach;
      __syncthreads();
      while (true) {
        const uint32_t grown = bg & (hdil3(sm.bits[1], wr - 1, wk) | hdil3(sm.bits[1], wr, wk) | hdil3(sm.bits[1], wr + 1, wk));
        const int changed = __syncthreads_or(grown != reach);
        reach = grown;
        sm.bits[1][wr][wk] = reach;
        __syncthreads();
        if (!changed) break;
      }
      sm.bits[0][wr][wk] = ~reach;
    }
    __syncthreads();
    // (4) binary_erosion(iterations=2) (utils.py:74)
    sm.bits[1][wr][wk] = erode_cross(sm.bits[0], wr, wk);
    __syncthreads();
    sm.bits[0][wr][wk] = erode_cross(sm.bits[1], wr, wk);
    __syncthreads();
    // (5) largest 4-connected component, first maximum wins (utils.py:75-79)
    for (int i = tid; i < T * T; i += NTHREADS) {
      sm.parent[i] = bit_at(sm.bits[0], i / T, i % T) ? (uint32_t)i : NONE;
      if ((i & 1) == 0) sm.area2[i >> 1] = 0;
    }
    if (tid == 0) { sm.best_key = 0; sm.min_root = NONE; }
    __syncthreads();
    for (int i = tid; i < T * T; i += NTHREADS) {
      if (sm.parent[i] == NONE) continue;
      const int r = i / T, c = i % T;
      if (c > 0 && bit_at(sm.bits[0], r, c - 1)) uf_union(sm.parent, i, i - 1);
      if (r > 0 && bit_at(sm.bits[0], r - 1, c)) uf_union(sm.parent, i, i - T);
    }
    __syncthreads();
    for (int i = tid; i < T * T; i += NTHREADS)
      if (sm.parent[i] != NONE) {
        const uint32_t root = uf_find(sm.parent, i);
        atomicAdd(&sm.area2[root >> 1], (root & 1u) ? 0x10000u : 1u);   // no carry between the halves: areas stay below 2^16
      }
    __syncthreads();
    for (int i = tid; i < T * T; i += NTHREADS)
      if (sm.parent[i] == (uint32_t)i) {
        const uint32_t area = (sm.area2[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu;
        atomicMax(&sm.best_key, (area << 14) | (uint32_t)(T * T - 1 - i));
      }
    __syncthreads();
    const bool any_region = sm.best_key != 0;
    if (any_region) {
      const uint32_t best_root = T * T - 1 - (sm.best_key & 0x3FFFu);
      uint32_t word = 0;
      for (int b = 0; b < 32; ++b) {
        const int i = wr * T + wk * 32 + b;
        if (sm.parent[i] != NONE && uf_find(sm.parent, i) == best_root) word |= 1u << b;
      }
      __syncthreads();
      sm.bits[0][wr][wk] = word;
      __syncthreads();
      // (6) binary_dilation(iterations=2) (utils.py:80)
      sm.bits[1][wr][wk] = dilate_cross(sm.bits[0], wr, wk);
      __syncthreads();
      sm.bits[0][wr][wk] = dilate_cross(sm.bits[1], wr, wk);
      __syncthreads();
    }
    // else: the (empty) label image itself is zoomed back (utils.py:75,81): all zero, bits[0] already is.

    // (7) up-scaling maps: which output rows / columns show which thumbnail row / column
    for (int i = tid; i < 2 * T; i += NTHREADS) {
      sm.first_o[i / T][i % T] = 1 << 30;
      sm.last_o[i / T][i % T] = -1;
    }
    __syncthreads();
    for (int o = tid; o < H; o += NTHREADS) {
      const int i = nn_index(up_y, o);
      if (i >= 0) { atomicMin(&sm.first_o[0][i], o); atomicMax(&sm.last_o[0][i], o); }
    }
    for (int o = tid; o < W; o += NTHREADS) {
      const int i = nn_index(up_x, o);
      if (i >= 0) { atomicMin(&sm.first_o[1][i], o); atomicMax(&sm.last_o[1][i], o); }
    }
    __syncthreads();
    if (tid < 2) {  // previous / next present index per axis (sequential, 128 steps)
      int prev = -1;
      for (int i = 0; i < T; ++i) {
        sm.prevp[tid][i] = (int16_t)prev;
        if (sm.last_o[tid][i] >= 0) prev = i;
      }
      int next = -1;
      for (int i = T - 1; i >= 0; --i) {
        sm.nextp[tid][i] = (int16_t)next;
        if (sm.last_o[tid][i] >= 0) next = i;
      }
    }
    __syncthreads();
    if (mask_out != nullptr) {  // utils.simple_bodymask's return value (only on request)
      uint8_t* mo = mask_out + (size_t)s * H * W;
      for (size_t p = tid; p < (size_t)H * W; p += NTHREADS) {
        const int oy = (int)(p / W), ox = (int)(p % W);
        const int iy = nn_index(up_y, oy), ix = nn_index(up_x, ox);
        mo[p] = (iy >= 0 && ix >= 0 && bit_at(sm.bits[0], iy, ix)) ? 1 : 0;
      }
    }
    // (8) bbox of label 1 of the 8-connected labelling of the up-scaled mask (utils.py:102-106), computed on
    // the PRESENT thumbnail rows / columns (the up-scaled mask is a block replication of that sub-grid).
    for (int i = tid; i < T * T; i += NTHREADS) {
      const int r = i / T, c = i % T;
      const bool on = sm.last_o[0][r] >= 0 && sm.last_o[1][c] >= 0 && bit_at(sm.bits[0], r, c);
      sm.parent[i] = on ? (uint32_t)i : NONE;
    }
    __syncthreads();
    for (int i = tid; i < T * T; i += NTHREADS) {
      if (sm.parent[i] == NONE) continue;
      const int r = i / T, c = i % T;
      const int pr = sm.prevp[0][r], pc = sm.prevp[1][c], nc = sm.nextp[1][c];
      if (pc >= 0 && sm.parent[r * T + pc] != NONE) uf_union(sm.parent, i, r * T + pc);
      if (pr >= 0) {
        if (sm.parent[pr * T + c] != NONE) uf_union(sm.parent, i, pr * T + c);
        if (pc >= 0 && sm.parent[pr * T + pc] != NONE) uf_union(sm.parent, i, pr * T + pc);
        if (nc >= 0 && sm.parent[pr * T + nc] != NONE) uf_union(sm.parent, i, pr * T + nc);
      }
    }
    if (tid == 0) { sm.bb[0] = 1 << 30; sm.bb[1] = 1 << 30; sm.bb[2] = -1; sm.bb[3] = -1; }
    __syncthreads();
    for (int i = tid; i < T * T; i += NTHREADS)
      if (sm.parent[i] == (uint32_t)i) atomicMin(&sm.min_root, (uint32_t)i);
    __syncthreads();
    const uint32_t root1 = sm.min_root;
    if (root1 != NONE) {
      for (int i = tid; i < T * T; i += NTHREADS) {
        if (sm.parent[i] == NONE || uf_find(sm.parent, i) != root1) continue;
        const int r = i / T, c = i % T;
        atomicMin(&sm.bb[0], (int)sm.first_o[0][r]);
        atomicMin(&sm.bb[1], (int)sm.first_o[1][c]);
        atomicMax(&sm.bb[2], (int)sm.last_o[0][r] + 1);
        atomicMax(&sm.bb[3], (int)sm.last_o[1][c] + 1);
      }
    }
    __syncthreads();
    if (tid == 0) {
      int32_t* b = boxes + 4 * s;
      if (root1 != NONE) { b[0] = sm.bb[0]; b[1] = sm.bb[1]; b[2] = sm.bb[2]; b[3] = sm.bb[3]; }
      else { b[0] = 0; b[1] = 0; b[2] = H; b[3] = W; }
    }
    __syncthreads();
  }
}

// zoom(crop, 256/crop.shape, order=1) on the clipped HU values, dtype preserved (utils.py:45,107-110).
// VT = int16: the result is rounded half away from zero to int16 (scipy's cast of an integer output array).
// VT = float / double (float volumes keep their dtype through the reference's pre-processing, utils.py:44-45,108-110):
// the interpolated value is cast to VT without rounding to an integer and then normalised as mask.py:167-168 does in
// that dtype - (x + 1024) / 1624 in float32 arithmetic for float32 volumes, in float64 for float64 - and stored as the
// fp32 the network receives (mask.py:178-182).
template <typename VT> struct ResizeOut { using type = float; };
template <> struct ResizeOut<int16_t> { using type = int16_t; };
template <typename VT>
__global__ void __launch_bounds__(256)
resize_kernel(const VT* __restrict__ vol, int S, int H, int W, const int32_t* __restrict__ boxes,
              typename ResizeOut<VT>::type* __restrict__ out, int OH, int OW, int clip) {
  const size_t total = (size_t)S * OH * OW;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int s = (int)(t / ((size_t)OH * OW));
    const int rem = (int)(t - (size_t)s * OH * OW);
    const int oy = rem / OW, ox = rem - oy * OW;
    const int32_t* b = boxes + 4 * s;
    const int r0 = b[0], c0 = b[1], h = b[2] - b[0], w = b[3] - b[1];
    const VT* img = vol + (size_t)s * H * W;
    const double sy = OH > 1 ? __ddiv_rn((double)(h - 1), (double)(OH - 1)) : 0.0;
    const double sx = OW > 1 ? __ddiv_rn((double)(w - 1), (double)(OW - 1)) : 0.0;
    const double ys = __dmul_rn((double)oy, sy), xs = __dmul_rn((double)ox, sx);
    double acc = 0.0;
    const bool inside = ys <= (double)(h - 1) && xs <= (double)(w - 1);
    if (inside) {
      const double fy0 = floor(ys), fx0 = floor(xs);
      const int y0 = (int)fy0, x0 = (int)fx0;
      const double fy = __dsub_rn(ys, fy0), fx = __dsub_rn(xs, fx0);
      const double wy[2] = {__dsub_rn(1.0, fy), fy}, wx[2] = {__dsub_rn(1.0, fx), fx};
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int yy = y0 + dy, xx = x0 + dx;
          double v = 0.0;
          if (yy < h && xx < w) {
            v = (double)img[(size_t)(r0 + yy) * W + (c0 + xx)];
            if (clip) v = v < -1024.0 ? -1024.0 : (v > 600.0 ? 600.0 : v);  // np.clip(-1024, 600), utils.py:45 (exact in every dtype)
          }
          acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(v, wy[dy]), wx[dx]));
        }
      }
    }
    if constexpr (sizeof(VT) == 2) {
      int16_t res = 0;
      if (inside) {
        acc = acc > 0.0 ? __dadd_rn(acc, 0.5) : __dsub_rn(acc, 0.5);  // scipy: round half away from zero
        double tr = trunc(acc);
        tr = tr < -32768.0 ? -32768.0 : (tr > 32767.0 ? 32767.0 : tr);
        res = (int16_t)tr;
      }
      out[t] = res;
    } else if constexpr (sizeof(VT) == 4) {
      float x = inside ? (float)acc : 0.f;                    // scipy casts the float64 sum to the float32 output array
      x = x > 600.f ? 600.f : x;                              // mask.py:167
      out[t] = __fdiv_rn(__fadd_rn(x, 1024.f), 1624.f);       // mask.py:168 in float32 (numpy keeps the array's dtype)
    } else {
      double x = inside ? acc : 0.0;
      x = x > 600.0 ? 600.0 : x;
      out[t] = (float)__ddiv_rn(__dadd_rn(x, 1024.0), 1624.0);  // float64 arithmetic, then the cast of mask.py:178-182
    }
  }
}

// Element conversion of orient_kernel.  Tin == Tout: the value itself.  Integer (and bool) elements into int16: clipped to
// [-1024, 600] first, as mask.py _to_int16_volume does on the host (the reference clips to that range before resampling
// and thresholds at -500 HU, so the clip changes no result).  Half-precision floats: widened to float32.
template <typename Tin, typename Tout>
struct Convert {
  static __device__ __forceinline__ Tout f(Tin x) {
    if constexpr (std::is_same<Tin, Tout>::value) {
      return x;
    } else if constexpr (std::is_same<Tout, int16_t>::value) {
      const long long v = (long long)x;
      return (int16_t)(v < -1024 ? -1024 : (v > 600 ? 600 : v));
    } else if constexpr (std::is_same<Tin, __half>::value) {
      return __half2float(x);
    } else {
      static_assert(std::is_same<Tin, __nv_bfloat16>::value && std::is_same<Tout, float>::value, "unsupported conversion");
      return __bfloat162float(x);
    }
  }
};

// Native orientation <-> LPS (OrientMap, preproc.cuh), every element passed through Convert<Tin, Tout>.
// to_lps != 0: threads walk the LPS array (coalesced writes) and gather; to_lps == 0: threads walk the native array
// (coalesced writes) and gather from the LPS array - the inverse map, orient_lps_of_native.  With the identity map the
// kernel is a plain conversion pass.
template <typename Tin, typename Tout>
__global__ void __launch_bounds__(256) orient_kernel(const Tin* __restrict__ src, Tout* __restrict__ dst, OrientMap m, int to_lps) {
  int dn[3];  // native dims: dn[perm[k]] = dl[k] (selects: a run-time index would put dn in local memory)
  for (int j = 0; j < 3; ++j) dn[j] = m.perm[0] == j ? m.dl[0] : (m.perm[1] == j ? m.dl[1] : m.dl[2]);
  const size_t n = (size_t)m.dl[0] * m.dl[1] * m.dl[2];
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    if (to_lps) {
      int i[3];
      i[2] = (int)(t % m.dl[2]);
      i[1] = (int)((t / m.dl[2]) % m.dl[1]);
      i[0] = (int)(t / ((size_t)m.dl[2] * m.dl[1]));
      int v[3], c[3];   // c[perm[k]] = v[k]
      for (int k = 0; k < 3; ++k) v[k] = m.flip[k] ? m.dl[k] - 1 - i[k] : i[k];
      for (int j = 0; j < 3; ++j) c[j] = m.perm[0] == j ? v[0] : (m.perm[1] == j ? v[1] : v[2]);
      dst[t] = Convert<Tin, Tout>::f(src[((size_t)c[0] * dn[1] + c[1]) * dn[2] + c[2]]);
    } else {
      int i[3];
      orient_lps_of_native(m, dn, t, i);
      dst[t] = Convert<Tin, Tout>::f(src[((size_t)i[0] * m.dl[1] + i[1]) * m.dl[2] + i[2]]);
    }
  }
}

}  // namespace

template <typename Tin, typename Tout = Tin>
static int launch_orient_t(const Tin* src, Tout* dst, const int dims_lps[3], const int perm[3], const int flip[3], int to_lps,
                           int num_sms, cudaStream_t stream) {
  OrientMap m;
  for (int k = 0; k < 3; ++k) { m.dl[k] = dims_lps[k]; m.perm[k] = perm[k]; m.flip[k] = flip[k]; }
  const size_t n = (size_t)dims_lps[0] * dims_lps[1] * dims_lps[2];
  size_t g = (n + 255) / 256;
  if (g > (size_t)num_sms * 16) g = (size_t)num_sms * 16;
  if (g < 1) g = 1;
  orient_kernel<Tin, Tout><<<(int)g, 256, 0, stream>>>(src, dst, m, to_lps);
  return (int)cudaGetLastError();
}
int launch_orient_convert(const void* src, int dtype, void* dst, const int dims_lps[3], const int perm[3], const int flip[3],
                          int num_sms, cudaStream_t stream) {
  int16_t* const d16 = static_cast<int16_t*>(dst);
  float* const d32 = static_cast<float*>(dst);
  switch (dtype) {
    case LM_DTYPE_I16: return launch_orient_t(static_cast<const int16_t*>(src), d16, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_F32: return launch_orient_t(static_cast<const float*>(src), d32, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_F64:
      return launch_orient_t(static_cast<const double*>(src), static_cast<double*>(dst), dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_U8: return launch_orient_t(static_cast<const uint8_t*>(src), d16, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_I8: return launch_orient_t(static_cast<const int8_t*>(src), d16, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_I32: return launch_orient_t(static_cast<const int32_t*>(src), d16, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_I64: return launch_orient_t(static_cast<const int64_t*>(src), d16, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_F16: return launch_orient_t(static_cast<const __half*>(src), d32, dims_lps, perm, flip, 1, num_sms, stream);
    case LM_DTYPE_BF16: return launch_orient_t(static_cast<const __nv_bfloat16*>(src), d32, dims_lps, perm, flip, 1, num_sms, stream);
    default: return -1;
  }
}
int launch_orient_u8(const uint8_t* src, uint8_t* dst, const int dims_lps[3], const int perm[3], const int flip[3], int to_lps,
                     int num_sms, cudaStream_t stream) {
  return launch_orient_t<uint8_t>(src, dst, dims_lps, perm, flip, to_lps, num_sms, stream);
}

int preproc_smem_bytes() { return (int)sizeof(Smem); }

template <typename VT>
static int launch_bodymask_t(const VT* vol, int S, int H, int W, int32_t* boxes, uint8_t* mask_out, int num_sms, cudaStream_t stream) {
  if (H < 1 || W < 1 || H > 16384 || W > 16384) return -10;
  static std::atomic<unsigned long long> attr_set_mask{0ull};  // engines of several host threads may launch concurrently  // the dynamic shared-memory opt-in is a per-device function attribute
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return -9;
  if (!((attr_set_mask.load(std::memory_order_acquire) >> dev) & 1ull)) {
    cudaError_t e = cudaFuncSetAttribute(bodymask_kernel<VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return (int)e;
    attr_set_mask.fetch_or(1ull << dev, std::memory_order_release);   // (benign race: setting the attribute twice is harmless)
  }
  const int grid = S < 2 * num_sms ? S : 2 * num_sms;
  bodymask_kernel<VT><<<grid, NTHREADS, sizeof(Smem), stream>>>(vol, S, H, W, boxes, mask_out);
  return (int)cudaGetLastError();
}
int launch_bodymask(const int16_t* vol, int S, int H, int W, int32_t* boxes, uint8_t* mask_out, int num_sms, cudaStream_t stream) {
  return launch_bodymask_t<int16_t>(vol, S, H, W, boxes, mask_out, num_sms, stream);
}
int launch_bodymask_float(const void* vol, int is_f64, int S, int H, int W, int32_t* boxes, uint8_t* mask_out, int num_sms,
                          cudaStream_t stream) {
  return is_f64 ? launch_bodymask_t<double>(static_cast<const double*>(vol), S, H, W, boxes, mask_out, num_sms, stream)
                : launch_bodymask_t<float>(static_cast<const float*>(vol), S, H, W, boxes, mask_out, num_sms, stream);
}

template <typename VT>
static int launch_resize_t(const VT* vol, int S, int H, int W, const int32_t* boxes, typename ResizeOut<VT>::type* out, int OH, int OW,
                           int clip, int num_sms, cudaStream_t stream) {
  const size_t total = (size_t)S * OH * OW;
  size_t g = (total + 255) / 256;
  if (g > (size_t)num_sms * 32) g = (size_t)num_sms * 32;
  resize_kernel<VT><<<(int)g, 256, 0, stream>>>(vol, S, H, W, boxes, out, OH, OW, clip);
  return (int)cudaGetLastError();
}
int launch_resize(const int16_t* vol, int S, int H, int W, const int32_t* boxes, int16_t* out, int OH, int OW, int clip,
                  int num_sms, cudaStream_t stream) {
  return launch_resize_t<int16_t>(vol, S, H, W, boxes, out, OH, OW, clip, num_sms, stream);
}
int launch_resize_float(const void* vol, int is_f64, int S, int H, int W, const int32_t* boxes, float* out_norm, int OH, int OW,
                        int num_sms, cudaStream_t stream) {
  return is_f64 ? launch_resize_t<double>(static_cast<const double*>(vol), S, H, W, boxes, out_norm, OH, OW, 1, num_sms, stream)
                : launch_resize_t<float>(static_cast<const float*>(vol), S, H, W, boxes, out_norm, OH, OW, 1, num_sms, stream);
}

}  // namespace lm
