// Mesh shape sums and maximum diameters of a label mask (lm_shape_sums_dev, lm_max_diameters_dev, DESIGN §4.10).
//
//   sums      one thread per 16 cubes along x: the four voxel rows of the cubes as 16-byte vectors plus one byte each.
//             A block of 16 cubes whose 68 labels are equal is skipped after one test; otherwise each mixed cube adds one
//             configuration per non-zero corner label, and the union configuration when a corner is 0.  Lanes holding
//             equal (row, configuration) keys add their count and corner sums once (__match_any_sync).  The rows "lung"
//             and 1..kSlots-1 are privatised in shared memory, the others go to global atomics.
//   moments   one thread per 16 voxels (mask_chunk.cuh): runs of one label within one x-row are summed in registers and
//             added once, privatised like the sums.
//   diameters (1) per axis-parallel line of every edge direction, the first and last vertex; (2) the vertices that are
//             first or last on their line along the axes of some diameter family, with a 3-bit extremality mask, and a
//             histogram of their planes per family; (3) on the host, the plane offsets; (4) the candidates scattered into
//             per-family plane buckets; (5) all pairs within each bucket, tiled through shared memory, one atomicMax of
//             the block's largest squared distance (a non-negative double, ordered as its bit pattern).
#include <math.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "mask_chunk.cuh"
#include "shape.cuh"

namespace lm {
namespace {

using u64 = unsigned long long;
constexpr int kThreads = 256;
constexpr int kSlots = 6;        // shared rows: slot 0 = "lung" (row 256), slot l = label l for l < kSlots
constexpr int kTile = kThreads;  // candidates per shared tile of the pair kernel
constexpr int kFamilies = 4;     // 3-D, equal axis 0, equal axis 1, equal axis 2
constexpr unsigned kFull = 0xffffffffu;

__host__ __device__ constexpr int family_bits(int f) { return f == 0 ? 7 : 7 & ~(1 << (f - 1)); }

__device__ __forceinline__ int slot_of(int row) { return row == 256 ? 0 : (row < kSlots ? row : -1); }

// ---- sums ---------------------------------------------------------------------------------------------------------
struct SumsDev {
  u64* counts;    // [257][256]
  u64* possum;    // [257][256][3]
  u64* moments;   // [257][10]
};

// 16 labels of row `row` (a flat voxel offset) from x = x0 on, 0 at or past n2; a 16-byte load when aligned and inside.
__device__ __forceinline__ uint4 row_chunk(const uint8_t* __restrict__ m, size_t row, int x0, int n2) {
  const uint8_t* p = m + row + x0;
  if (x0 + kChunk <= n2 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) return __ldg(reinterpret_cast<const uint4*>(p));
  unsigned w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < kChunk; ++k)
    if (x0 + k < n2) w[k >> 2] |= (unsigned)p[k] << (8 * (k & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Sum over the lanes of `peers` of v (0 .. 2^32 - 1), exact: 16-bit halves through the 32-bit reduction.
__device__ __forceinline__ u64 peer_sum(unsigned peers, unsigned v) {
  const unsigned lo = __reduce_add_sync(peers, v & 0xffffu), hi = __reduce_add_sync(peers, v >> 16);
  return ((u64)hi << 16) + lo;
}

__device__ __forceinline__ void add_cube(int row, int conf, int p0, int p1, int p2, u64* s_cnt, u64* s_pos, const SumsDev& g) {
  const int key = row * 256 + conf;
  const unsigned peers = __match_any_sync(__activemask(), key);
  const unsigned n = __popc(peers);
  // p + 1 >= 0, so the sums are taken of p + 1 and n is subtracted
  const u64 q0 = peer_sum(peers, (unsigned)(p0 + 1)) - n, q1 = peer_sum(peers, (unsigned)(p1 + 1)) - n,
            q2 = peer_sum(peers, (unsigned)(p2 + 1)) - n;
  if ((int)(threadIdx.x & 31) != __ffs(peers) - 1) return;
  const int s = slot_of(row);
  u64* c = s >= 0 ? &s_cnt[s * 256 + conf] : &g.counts[key];
  u64* q = s >= 0 ? &s_pos[(s * 256 + conf) * 3] : &g.possum[(size_t)key * 3];
  atomicAdd(c, (u64)n);
  atomicAdd(q, q0);
  atomicAdd(q + 1, q1);
  atomicAdd(q + 2, q2);
}

__global__ void __launch_bounds__(kThreads) shape_cubes_kernel(const uint8_t* __restrict__ mask, int n0, int n1, int n2,
                                                              SumsDev g) {
  __shared__ u64 s_cnt[kSlots * 256], s_pos[kSlots * 256 * 3];
  for (int i = threadIdx.x; i < kSlots * 256; i += blockDim.x) s_cnt[i] = 0;
  for (int i = threadIdx.x; i < kSlots * 256 * 3; i += blockDim.x) s_pos[i] = 0;
  __syncthreads();
  const int chunks = (n2 + 1 + kChunk - 1) / kChunk;   // chunk c: cubes p2 = 16c - 1 .. 16c + 14
  const size_t items = (size_t)(n0 + 1) * (n1 + 1) * chunks;
  for (size_t it = blockIdx.x * (size_t)blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(it % chunks);
    const size_t pl = it / chunks;
    const int p1 = (int)(pl % (n1 + 1)) - 1, p0 = (int)(pl / (n1 + 1)) - 1;
    const int x0 = c * kChunk;
    uint4 v[4];
    int e[4];   // the label at x0 - 1
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int q0 = p0 + (r >> 1), q1 = p1 + (r & 1);
      if (q0 < 0 || q0 >= n0 || q1 < 0 || q1 >= n1) {
        v[r] = make_uint4(0, 0, 0, 0);
        e[r] = 0;
      } else {
        const size_t row = ((size_t)q0 * n1 + q1) * n2;
        v[r] = row_chunk(mask, row, x0, n2);
        e[r] = x0 > 0 ? mask[row + x0 - 1] : 0;
      }
    }
    const unsigned rep = (unsigned)e[0] * 0x01010101u;
    bool uniform = true;
#pragma unroll
    for (int r = 0; r < 4; ++r)
      uniform = uniform && e[r] == e[0] && v[r].x == rep && v[r].y == rep && v[r].z == rep && v[r].w == rep;
    if (uniform) continue;
#pragma unroll
    for (int t = 0; t < kChunk; ++t) {
      int lab[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int r = k >> 1;   // (d0, d1) = (k >> 2, (k >> 1) & 1)
        lab[k] = (k & 1) ? label_at(v[r], t) : (t == 0 ? e[r] : label_at(v[r], t - 1));
      }
      bool same = true;
#pragma unroll
      for (int k = 1; k < 8; ++k) same = same && lab[k] == lab[0];
      if (same) continue;
      const int p2 = x0 - 1 + t;
      unsigned done = 0, zero = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) zero |= (lab[k] == 0 ? 1u : 0u) << k;
      done = zero;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (done & (1u << k)) continue;
        unsigned conf = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) conf |= (lab[q] == lab[k] ? 1u : 0u) << q;
        done |= conf;
        add_cube(lab[k], (int)conf, p0, p1, p2, s_cnt, s_pos, g);
      }
      if (zero) add_cube(256, (int)(~zero & 255u), p0, p1, p2, s_cnt, s_pos, g);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSlots * 256; i += blockDim.x) {
    if (!s_cnt[i]) continue;
    const int s = i >> 8, row = s == 0 ? 256 : s;
    const size_t key = (size_t)row * 256 + (i & 255);
    atomicAdd(&g.counts[key], s_cnt[i]);
    for (int a = 0; a < 3; ++a) atomicAdd(&g.possum[key * 3 + a], s_pos[i * 3 + a]);
  }
}

// A run of `c` voxels of `row` in x-row (i, j) with index sums sk, skk: its 10 moments.
__device__ __forceinline__ void add_run(int row, u64 i, u64 j, u64 c, u64 sk, u64 skk, u64* s_mom, const SumsDev& g) {
  const int s = slot_of(row);
  u64* m = s >= 0 ? &s_mom[s * kShapeMoments] : &g.moments[(size_t)row * kShapeMoments];
  const u64 v[kShapeMoments] = {c, i * c, j * c, sk, i * i * c, j * j * c, skk, i * j * c, i * sk, j * sk};
#pragma unroll
  for (int k = 0; k < kShapeMoments; ++k)
    if (v[k]) atomicAdd(&m[k], v[k]);
}

__global__ void __launch_bounds__(kThreads) shape_moments_kernel(const uint8_t* __restrict__ mask, int n1, int n2, size_t n,
                                                                SumsDev g) {
  __shared__ u64 s_mom[kSlots * kShapeMoments];
  for (int i = threadIdx.x; i < kSlots * kShapeMoments; i += blockDim.x) s_mom[i] = 0;
  __syncthreads();
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    if ((lab.x | lab.y | lab.z | lab.w) == 0) continue;
    u64 k = base % n2, line = base / n2, j = line % n1, i = line / n1;
    int run = 0;              // the label of the current run (0: none)
    u64 rc = 0, rk = 0, rkk = 0, uc = 0, uk = 0, ukk = 0;   // the run's and the union run's count, sum k, sum k^2
    for (int t = 0; t < kChunk && base + t < n; ++t) {
      const int l = label_at(lab, t);
      if (l != run) {
        if (run) add_run(run, i, j, rc, rk, rkk, s_mom, g);
        run = l;
        rc = rk = rkk = 0;
      }
      if (!l && uc) {
        add_run(256, i, j, uc, uk, ukk, s_mom, g);
        uc = uk = ukk = 0;
      }
      if (l) {
        ++rc; rk += k; rkk += k * k;
        ++uc; uk += k; ukk += k * k;
      }
      if (++k == (u64)n2) {   // the next voxel starts a new x-row: close both runs
        if (run) add_run(run, i, j, rc, rk, rkk, s_mom, g);
        if (uc) add_run(256, i, j, uc, uk, ukk, s_mom, g);
        run = 0;
        rc = rk = rkk = uc = uk = ukk = 0;
        k = 0;
        if (++j == (u64)n1) { j = 0; ++i; }
      }
    }
    if (run) add_run(run, i, j, rc, rk, rkk, s_mom, g);
    if (uc) add_run(256, i, j, uc, uk, ukk, s_mom, g);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kSlots * kShapeMoments; t += blockDim.x) {
    const int s = t / kShapeMoments, row = s == 0 ? 256 : s;
    if (s_mom[t]) atomicAdd(&g.moments[(size_t)row * kShapeMoments + t % kShapeMoments], s_mom[t]);
  }
}

// ---- diameters ----------------------------------------------------------------------------------------------------
// Edge direction k: the node u (its lower end) has u_k in -1..n_k-1 and u_m in 0..n_m-1 (m != k), stored at index
// i_m = u_m + (m == k) of a grid N_m = n_m + (m == k).  Its vertex has doubled coordinates c_m = 2 u_m + (m == k) =
// 2 i_m - (m == k).  The
// line of (k, j) through a node fixes i_a, i_b (a < b, both != j): index i_a * N_b + i_b of table (k, j).
struct Geo {
  int n[3];
  int row;
  size_t off[9];     // first line of table (k, j) at k * 3 + j
};

template <int K>
__device__ __forceinline__ int nk(const Geo& g, int m) { return g.n[m] + (m == K); }

__device__ __forceinline__ bool member(const uint8_t* __restrict__ mask, const Geo& g, int v0, int v1, int v2) {
  if (v0 < 0 || v0 >= g.n[0] || v1 < 0 || v1 >= g.n[1] || v2 < 0 || v2 >= g.n[2]) return false;
  const int l = mask[((size_t)v0 * g.n[1] + v1) * g.n[2] + v2];
  return g.row == 256 ? l != 0 : l == g.row;
}

// Is there a vertex on the K-edge of node index (i0, i1, i2)?
template <int K>
__device__ __forceinline__ bool crossing(const uint8_t* __restrict__ mask, const Geo& g, int i0, int i1, int i2) {
  const int u0 = i0 - (K == 0), u1 = i1 - (K == 1), u2 = i2 - (K == 2);
  return member(mask, g, u0, u1, u2) != member(mask, g, u0 + (K == 0), u1 + (K == 1), u2 + (K == 2));
}

// The axes a < b other than j.
__host__ __device__ constexpr int axis_a(int j) { return j == 0 ? 1 : 0; }
__host__ __device__ constexpr int axis_b(int j) { return j == 2 ? 1 : 2; }

// Table (K, J): one thread per line, the first and last node index along J with a vertex (-1, -1 without one).
template <int K, int J>
__global__ void __launch_bounds__(kThreads) line_ends_kernel(const uint8_t* __restrict__ mask, Geo g, size_t lines,
                                                             int2* __restrict__ tab) {
  constexpr int A = axis_a(J), B = axis_b(J);
  for (size_t L = blockIdx.x * (size_t)blockDim.x + threadIdx.x; L < lines; L += (size_t)gridDim.x * blockDim.x) {
    const int ia = (int)(L / nk<K>(g, B)), ib = (int)(L % nk<K>(g, B));
    int first = -1, last = -1;
    const int len = nk<K>(g, J);
    for (int t = 0; t < len; ++t) {
      const int i0 = J == 0 ? t : ia, i1 = J == 1 ? t : (A == 1 ? ia : ib), i2 = J == 2 ? t : ib;
      if (crossing<K>(mask, g, i0, i1, i2)) {
        if (first < 0) first = t;
        last = t;
      }
    }
    tab[g.off[K * 3 + J] + L] = make_int2(first, last);
  }
}

// Plane index of a candidate in family f (f >= 1): its doubled coordinate along axis f - 1, plus 1.
__device__ __forceinline__ int plane_of(const int4& c, int f) { return (f == 1 ? c.x : (f == 2 ? c.y : c.z)) + 1; }

struct CandDev {
  int4* cand;                 // (c0, c1, c2, extremality bits)
  unsigned* n_cand;
  unsigned* hist[kFamilies];  // planes per family: 1, 2 n0 + 1, 2 n1 + 1, 2 n2 + 1
  size_t cap;
};

template <int K, int J>
__device__ __forceinline__ bool line_end(const Geo& g, const int2* __restrict__ tab, int i0, int i1, int i2) {
  constexpr int A = axis_a(J), B = axis_b(J);
  const int i[3] = {i0, i1, i2};
  const int2 fl = tab[g.off[K * 3 + J] + (size_t)i[A] * nk<K>(g, B) + i[B]];
  return i[J] == fl.x || i[J] == fl.y;
}

// Every K-edge node with a vertex: its extremality bits (bit j: first or last on its line along j); the vertices some
// diameter family needs are appended with their bits and counted in the family's plane histogram.
template <int K>
__global__ void __launch_bounds__(kThreads) candidates_kernel(const uint8_t* __restrict__ mask, Geo g,
                                                             const int2* __restrict__ tab, CandDev cd, unsigned* overflow) {
  const size_t total = (size_t)nk<K>(g, 0) * nk<K>(g, 1) * nk<K>(g, 2);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int i2 = (int)(t % nk<K>(g, 2));
    const size_t r = t / nk<K>(g, 2);
    const int i1 = (int)(r % nk<K>(g, 1)), i0 = (int)(r / nk<K>(g, 1));
    if (!crossing<K>(mask, g, i0, i1, i2)) continue;
    const unsigned bits = (line_end<K, 0>(g, tab, i0, i1, i2) ? 1u : 0u) | (line_end<K, 1>(g, tab, i0, i1, i2) ? 2u : 0u) |
                          (line_end<K, 2>(g, tab, i0, i1, i2) ? 4u : 0u);
    bool keep = false;
#pragma unroll
    for (int f = 0; f < kFamilies; ++f) keep = keep || (bits & family_bits(f)) == (unsigned)family_bits(f);
    if (!keep) continue;
    const int4 c = make_int4(2 * i0 - (K == 0), 2 * i1 - (K == 1), 2 * i2 - (K == 2), (int)bits);
    const unsigned pos = atomicAdd(cd.n_cand, 1u);
    if (pos >= cd.cap) { atomicOr(overflow, 1u); continue; }
    cd.cand[pos] = c;
#pragma unroll
    for (int f = 0; f < kFamilies; ++f)
      if ((bits & family_bits(f)) == (unsigned)family_bits(f)) atomicAdd(&cd.hist[f][f == 0 ? 0 : plane_of(c, f)], 1u);
  }
}

struct Buckets {
  int4* pts[kFamilies];        // each family's candidates, bucketed by plane
  unsigned* cursor[kFamilies]; // the next free slot of each plane (starts at the plane's offset)
};

__global__ void __launch_bounds__(kThreads) scatter_kernel(const int4* __restrict__ cand, unsigned n, Buckets bk) {
  for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const int4 c = cand[t];
#pragma unroll
    for (int f = 0; f < kFamilies; ++f)
      if (((unsigned)c.w & family_bits(f)) == (unsigned)family_bits(f))
        bk.pts[f][atomicAdd(&bk.cursor[f][f == 0 ? 0 : plane_of(c, f)], 1u)] = c;
  }
}

// d^2 = ((D2 h2)^2 + (D1 h1)^2) + (D0 h0)^2, every operation rounded on its own (the order of lm_surface_distance_dev).
__device__ __forceinline__ double dist2(int4 a, int b0, int b1, int b2, double h0, double h1, double h2) {
  const double t0 = __dmul_rn((double)(a.x - b0), h0), t1 = __dmul_rn((double)(a.y - b1), h1),
               t2 = __dmul_rn((double)(a.z - b2), h2);
  return __dadd_rn(__dadd_rn(__dmul_rn(t2, t2), __dmul_rn(t1, t1)), __dmul_rn(t0, t0));
}

// All pairs within each segment [off[s], off[s + 1]) of pts (blockIdx.y strides over the segments); the largest d^2 goes
// to *out as its bit pattern.
__global__ void __launch_bounds__(kThreads) pair_max_kernel(const int4* __restrict__ pts, const unsigned* __restrict__ off,
                                                           int segs, double h0, double h1, double h2, u64* out) {
  __shared__ int s0[kTile], s1[kTile], s2[kTile];
  __shared__ double s_max[kThreads / 32];
  double best = 0.0;
  for (int s = blockIdx.y; s < segs; s += gridDim.y) {
    const unsigned begin = off[s], len = off[s + 1] - begin;
    if (len < 2) continue;   // block-uniform
    const unsigned T = (len + kTile - 1) / kTile;
    const unsigned long long pairs = (unsigned long long)T * (T + 1) / 2;
    for (unsigned long long tp = blockIdx.x; tp < pairs; tp += gridDim.x) {
      unsigned ti = 0;
      unsigned long long rem = tp;
      while (rem >= T - ti) { rem -= T - ti; ++ti; }
      const unsigned tj = ti + (unsigned)rem;
      __syncthreads();
      const unsigned jb = tj * kTile, jn = min((unsigned)kTile, len - jb);
      if (threadIdx.x < jn) {
        const int4 c = pts[begin + jb + threadIdx.x];
        s0[threadIdx.x] = c.x; s1[threadIdx.x] = c.y; s2[threadIdx.x] = c.z;
      }
      __syncthreads();
      const unsigned i = ti * kTile + threadIdx.x;
      if (i < len) {
        const int4 a = pts[begin + i];
        for (unsigned q = 0; q < jn; ++q) best = fmax(best, dist2(a, s0[q], s1[q], s2[q], h0, h1, h2));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(kFull, best, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) best = fmax(best, s_max[w]);
    if (best > 0.0) atomicMax(out, (u64)__double_as_longlong(best));
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
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

size_t table_lines(const int* n, int k, int j) {
  size_t l = 1;
  for (int m = 0; m < 3; ++m)
    if (m != j) l *= (size_t)(n[m] + (m == k));
  return l;
}

}  // namespace

int ShapeWork::reserve(size_t bytes, size_t f_need) {
  if (bytes > d_bytes) {
    if (d) cudaFree(d);
    d = nullptr;
    d_bytes = 0;
    SC(cudaMalloc(&d, bytes));
    d_bytes = bytes;
  }
  if (f_need > f_bytes) {
    if (f) cudaFree(f);
    f = nullptr;
    f_bytes = 0;
    SC(cudaMalloc(&f, f_need));
    f_bytes = f_need;
  }
  return 0;
}

void ShapeWork::release() {
  if (d) cudaFree(d);
  if (f) cudaFree(f);
  d = f = nullptr;
  d_bytes = f_bytes = 0;
}

int shape_sums(ShapeWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int64_t* counts, int64_t* possum, int64_t* moments,
               int num_sms, cudaStream_t st, int64_t* launches) {
  const size_t nc = (size_t)kShapeRows * 256, np3 = nc * 3, nm = (size_t)kShapeRows * kShapeMoments;
  const size_t bytes = (nc + np3 + nm) * sizeof(u64);
  SC((cudaError_t)w.reserve(bytes, 0));
  SumsDev g{static_cast<u64*>(w.d), static_cast<u64*>(w.d) + nc, static_cast<u64*>(w.d) + nc + np3};
  SC(cudaMemsetAsync(w.d, 0, bytes, st));
  const size_t items = (size_t)(n0 + 1) * (n1 + 1) * ((n2 + kChunk) / kChunk);
  shape_cubes_kernel<<<grid_for(shape_cubes_kernel, items, num_sms), kThreads, 0, st>>>(d_mask, n0, n1, n2, g);
  SC(cudaGetLastError());
  const size_t n = (size_t)n0 * n1 * n2;
  shape_moments_kernel<<<grid_for(shape_moments_kernel, (n + kChunk - 1) / kChunk, num_sms), kThreads, 0, st>>>(d_mask, n1, n2,
                                                                                                                n, g);
  SC(cudaGetLastError());
  *launches += 2;
  SC(cudaMemcpyAsync(counts, g.counts, nc * sizeof(u64), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(possum, g.possum, np3 * sizeof(u64), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(moments, g.moments, nm * sizeof(u64), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  return 0;
}

int max_diameters(ShapeWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const double* spacing, double* d2,
                  int num_sms, cudaStream_t st, int64_t* launches) {
  Geo g{};
  g.n[0] = n0; g.n[1] = n1; g.n[2] = n2;
  g.row = row;
  size_t lines = 0, along01 = 0;
  for (int kj = 0; kj < 9; ++kj) {
    g.off[kj] = lines;
    const size_t l = table_lines(g.n, kj / 3, kj % 3);
    lines += l;
    if (kj % 3 < 2) along01 += l;
  }
  // Every candidate is first or last on its line along axis 0 or axis 1 (each family needs one of the two).
  const size_t cap = 2 * along01;
  size_t planes[kFamilies] = {1, 2 * (size_t)n0 + 1, 2 * (size_t)n1 + 1, 2 * (size_t)n2 + 1}, all_planes = 0;
  for (int f = 0; f < kFamilies; ++f) all_planes += planes[f];
  // d: squared diameters [4] | overflow flag | candidate count | histograms | line tables | candidates
  const size_t o_flag = align256(kFamilies * sizeof(u64)), o_n = o_flag + 256, o_hist = o_n + 256;
  const size_t o_tab = o_hist + align256(all_planes * sizeof(unsigned)), o_cand = o_tab + align256(lines * sizeof(int2));
  const size_t bytes = o_cand + cap * sizeof(int4);
  SC((cudaError_t)w.reserve(bytes, 0));
  char* base = static_cast<char*>(w.d);
  u64* d_d2 = reinterpret_cast<u64*>(base);
  unsigned* d_flag = reinterpret_cast<unsigned*>(base + o_flag);
  CandDev cd{reinterpret_cast<int4*>(base + o_cand), reinterpret_cast<unsigned*>(base + o_n), {}, cap};
  size_t at = 0;
  for (int f = 0; f < kFamilies; ++f) {
    cd.hist[f] = reinterpret_cast<unsigned*>(base + o_hist) + at;
    at += planes[f];
  }
  SC(cudaMemsetAsync(base, 0, o_tab, st));
  int2* tab = reinterpret_cast<int2*>(base + o_tab);
#define LM_LINES(K, J)                                                                                                   \
  do {                                                                                                                   \
    const size_t l_ = table_lines(g.n, K, J);                                                                            \
    line_ends_kernel<K, J><<<grid_for(line_ends_kernel<K, J>, l_, num_sms), kThreads, 0, st>>>(d_mask, g, l_, tab);      \
    SC(cudaGetLastError());                                                                                              \
  } while (0)
  LM_LINES(0, 0); LM_LINES(0, 1); LM_LINES(0, 2);
  LM_LINES(1, 0); LM_LINES(1, 1); LM_LINES(1, 2);
  LM_LINES(2, 0); LM_LINES(2, 1); LM_LINES(2, 2);
#undef LM_LINES
  candidates_kernel<0><<<grid_for(candidates_kernel<0>, (size_t)(n0 + 1) * n1 * n2, num_sms), kThreads, 0, st>>>(d_mask, g, tab, cd, d_flag);
  candidates_kernel<1><<<grid_for(candidates_kernel<1>, (size_t)n0 * (n1 + 1) * n2, num_sms), kThreads, 0, st>>>(d_mask, g, tab, cd, d_flag);
  candidates_kernel<2><<<grid_for(candidates_kernel<2>, (size_t)n0 * n1 * (n2 + 1), num_sms), kThreads, 0, st>>>(d_mask, g, tab, cd, d_flag);
  SC(cudaGetLastError());
  *launches += 12;
  // the plane histograms -> per-family bucket offsets
  std::vector<unsigned> hist(all_planes + 2);
  SC(cudaMemcpyAsync(hist.data(), cd.hist[0], all_planes * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(&hist[all_planes], cd.n_cand, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(&hist[all_planes + 1], d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  if (hist[all_planes + 1]) return -1;   // cannot happen: cap bounds the candidates
  const unsigned n_cand = hist[all_planes];
  std::vector<unsigned> offs(all_planes + kFamilies);   // family f: planes[f] + 1 offsets into its own bucket array
  size_t fam_at[kFamilies], pts = 0, h = 0, o = 0;
  for (int f = 0; f < kFamilies; ++f) {
    fam_at[f] = o;
    unsigned run = 0;
    for (size_t p = 0; p < planes[f]; ++p) {
      offs[o++] = run;
      run += hist[h++];
    }
    offs[o++] = run;
    pts += run;
  }
  const size_t o_pts = align256(offs.size() * sizeof(unsigned) * 2);
  SC((cudaError_t)w.reserve(bytes, o_pts + std::max<size_t>(pts, 1) * sizeof(int4)));
  char* fb = static_cast<char*>(w.f);
  unsigned* d_offs = reinterpret_cast<unsigned*>(fb);
  unsigned* d_cursor = d_offs + offs.size();
  SC(cudaMemcpyAsync(d_offs, offs.data(), offs.size() * sizeof(unsigned), cudaMemcpyHostToDevice, st));
  SC(cudaMemcpyAsync(d_cursor, offs.data(), offs.size() * sizeof(unsigned), cudaMemcpyHostToDevice, st));
  Buckets bk{};
  size_t pts_at = 0;
  for (int f = 0; f < kFamilies; ++f) {
    bk.pts[f] = reinterpret_cast<int4*>(fb + o_pts) + pts_at;
    bk.cursor[f] = d_cursor + fam_at[f];
    pts_at += offs[fam_at[f] + planes[f]];
  }
  if (n_cand) {
    scatter_kernel<<<grid_for(scatter_kernel, n_cand, num_sms), kThreads, 0, st>>>(cd.cand, n_cand, bk);
    SC(cudaGetLastError());
    ++*launches;
  }
  const double h0 = spacing[0] * 0.5, h1 = spacing[1] * 0.5, h2 = spacing[2] * 0.5;
  for (int f = 0; f < kFamilies; ++f) {
    const unsigned fam_n = offs[fam_at[f] + planes[f]];
    if (fam_n < 2) continue;
    const unsigned long long tiles = (fam_n + kTile - 1) / kTile;
    dim3 grid;
    if (f == 0) {
      grid = dim3((unsigned)std::min<unsigned long long>(tiles * (tiles + 1) / 2, (unsigned long long)num_sms * 16), 1);
    } else {
      grid = dim3(4, (unsigned)std::min<size_t>(planes[f], 65535));
    }
    pair_max_kernel<<<grid, kThreads, 0, st>>>(bk.pts[f], d_offs + fam_at[f], (int)planes[f], h0, h1, h2, d_d2 + f);
    SC(cudaGetLastError());
    ++*launches;
  }
  u64 out[kFamilies];
  SC(cudaMemcpyAsync(out, d_d2, sizeof(out), cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  for (int f = 0; f < kFamilies; ++f) memcpy(&d2[f], &out[f], sizeof(double));
  return 0;
}

}  // namespace lm
