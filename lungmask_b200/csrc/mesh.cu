// Marching-cubes surface meshes of one row of a label mask (lm_mesh_counts_dev, lm_mesh_emit_dev, DESIGN §4.14).
//
//   lines   the padded grid's points q with a vertex have q0 in -1..n0-1 and q1 in -1..n1-1, as do the cubes' lowest
//           corners p; line (a, b) holds q0 = a - 1, q1 = b - 1 and x = q2 = -1..n2-1, lines in row-major order, so the
//           padded linear order of the points (and of the cubes) is line order, then x.  One warp per line walks x in
//           chunks of 32 (lane = x - chunk start); a lane reads each row's label at x and takes x + 1 from the next lane.
//   count   per line: V = the crossing edges (q, m) of its points, T = the triangles of its cubes' configurations.
//   scan    the per-line (V, T) are scanned in place to exclusive offsets per segment of kSegment lines, plus the
//           segments' offsets and the totals.
//   emit    the same walk over the rows of the four lines (q0 + d0, q1 + d1), d0, d1 in {0, 1}: every lane gets, for each
//           of them, its vertex bits at x and the number of vertices before x (ballots), so that an edge (a, m) of cube
//           p names vertex (p + corner a, m) by offset arithmetic.  The line's own vertices and its cubes' triangles
//           (table order) are written at their offsets; nothing is sorted.
//   A chunk whose cubes are all inside or all outside the row (in the four lines the walk reads) is skipped after one
//   vote.
#include <math.h>

#include <algorithm>

#include "mesh.cuh"

namespace lm {
namespace {

using u64 = unsigned long long;
constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kScanThreads = 1024, kScanItems = 8, kSegment = kScanThreads * kScanItems;

struct MeshGeo {
  int n0, n1, n2, row;
};

__device__ __forceinline__ unsigned member(const uint8_t* __restrict__ m, const MeshGeo& g, int q0, int q1, int x) {
  if (q0 < 0 || q0 >= g.n0 || q1 < 0 || q1 >= g.n1 || x < 0 || x >= g.n2) return 0u;
  const int l = m[((size_t)q0 * g.n1 + q1) * g.n2 + x];
  return (g.row == 256 ? l != 0 : l == g.row) ? 1u : 0u;
}

// Membership of row (q0, q1) at the lane's x (bit 0) and at x + 1 (bit 1).
__device__ __forceinline__ unsigned member_pair(const uint8_t* __restrict__ m, const MeshGeo& g, int q0, int q1, int x,
                                                int lane) {
  const unsigned h = member(m, g, q0, q1, x);
  unsigned n = __shfl_down_sync(kFull, h, 1);
  if (lane == 31) n = member(m, g, q0, q1, x + 1);
  return h | (n << 1);
}

// Configuration of the cube at (q0, q1, x) from the pairs of rows (q0 + d0, q1 + d1): bit k is corner
// ((k >> 2) & 1, (k >> 1) & 1, k & 1).
__device__ __forceinline__ unsigned cube_config(unsigned r00, unsigned r01, unsigned r10, unsigned r11) {
  return r00 | (r01 << 2) | (r10 << 4) | (r11 << 6);
}

// Vertex bits at x of a line from its row pair r and the pairs of the rows one step along axis 0 (r0) and axis 1 (r1).
__device__ __forceinline__ unsigned vertex_bits(unsigned r, unsigned r0, unsigned r1) {
  return ((r ^ r0) & 1u) | (((r ^ r1) & 1u) << 1) | (((r ^ (r >> 1)) & 1u) << 2);
}

__device__ __forceinline__ u64 warp_sum(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads) mesh_count_kernel(const uint8_t* __restrict__ mask, MeshGeo g,
                                                             const int32_t* __restrict__ t_off, size_t lines,
                                                             u64* __restrict__ cnt_v, u64* __restrict__ cnt_t) {
  __shared__ uint8_t s_ntri[kMeshConfigs];
  for (int i = threadIdx.x; i < kMeshConfigs; i += blockDim.x) s_ntri[i] = (uint8_t)(t_off[i + 1] - t_off[i]);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t L = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; L < lines; L += warps) {
    const int q0 = (int)(L / (g.n1 + 1)) - 1, q1 = (int)(L % (g.n1 + 1)) - 1;
    unsigned v = 0, t = 0;   // this lane's share: at most 5 per chunk
    for (int x0 = -1; x0 < g.n2; x0 += 32) {
      const int x = x0 + lane;
      const unsigned r00 = member_pair(mask, g, q0, q1, x, lane), r01 = member_pair(mask, g, q0, q1 + 1, x, lane),
                     r10 = member_pair(mask, g, q0 + 1, q1, x, lane), r11 = member_pair(mask, g, q0 + 1, q1 + 1, x, lane);
      const unsigned c = cube_config(r00, r01, r10, r11);
      if (__all_sync(kFull, c == 0u || c == 255u)) continue;
      v += __popc(vertex_bits(r00, r10, r01));
      t += s_ntri[c];
    }
    const u64 sv = warp_sum(v), st = warp_sum(t);
    if (lane == 0) {
      cnt_v[L] = sv;
      cnt_t[L] = st;
    }
  }
}

// Exclusive scan of one value per thread over the block; *total gets the block's sum.  s: 32 words of shared memory.
__device__ __forceinline__ u64 block_exclusive(u64 v, u64* s, u64* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  u64 inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 y = __shfl_up_sync(kFull, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    u64 w = lane < (int)(blockDim.x >> 5) ? s[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 y = __shfl_up_sync(kFull, w, o);
      if (lane >= o) w += y;
    }
    s[lane] = w;
  }
  __syncthreads();
  const u64 before = wid ? s[wid - 1] : 0;
  *total = s[31];
  __syncthreads();
  return before + inc - v;
}

// Per segment of kSegment lines: the exclusive offsets in place, the segment's totals to seg_v / seg_t.
__global__ void __launch_bounds__(kScanThreads) mesh_scan_kernel(u64* __restrict__ cnt_v, u64* __restrict__ cnt_t,
                                                                size_t lines, u64* __restrict__ seg_v,
                                                                u64* __restrict__ seg_t) {
  __shared__ u64 s_v[32], s_t[32];
  const size_t base = (size_t)blockIdx.x * kSegment + (size_t)threadIdx.x * kScanItems;
  u64 v[kScanItems], t[kScanItems], sv = 0, st = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = base + k < lines ? cnt_v[base + k] : 0;
    t[k] = base + k < lines ? cnt_t[base + k] : 0;
    sv += v[k];
    st += t[k];
  }
  u64 tot_v, tot_t;
  u64 ev = block_exclusive(sv, s_v, &tot_v), et = block_exclusive(st, s_t, &tot_t);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < lines) {
      cnt_v[base + k] = ev;
      cnt_t[base + k] = et;
    }
    ev += v[k];
    et += t[k];
  }
  if (threadIdx.x == 0) {
    seg_v[blockIdx.x] = tot_v;
    seg_t[blockIdx.x] = tot_t;
  }
}

// One block: the segments' exclusive offsets in place, the totals at [segs].
__global__ void __launch_bounds__(kScanThreads) mesh_scan_top_kernel(u64* __restrict__ seg_v, u64* __restrict__ seg_t,
                                                                    int segs) {
  __shared__ u64 s_v[32], s_t[32];
  u64 carry_v = 0, carry_t = 0;
  for (int b = 0; b < segs; b += kScanThreads) {
    const int i = b + threadIdx.x;
    const u64 v = i < segs ? seg_v[i] : 0, t = i < segs ? seg_t[i] : 0;
    u64 tot_v, tot_t;
    const u64 ev = block_exclusive(v, s_v, &tot_v), et = block_exclusive(t, s_t, &tot_t);
    if (i < segs) {
      seg_v[i] = carry_v + ev;
      seg_t[i] = carry_t + et;
    }
    carry_v += tot_v;
    carry_t += tot_t;
  }
  if (threadIdx.x == 0) {
    seg_v[segs] = carry_v;
    seg_t[segs] = carry_t;
  }
}

struct Offsets {
  const u64* line_v;   // exclusive within the line's segment
  const u64* line_t;
  const u64* seg_v;    // the segments' offsets
  const u64* seg_t;
};

__device__ __forceinline__ u64 line_vertex_offset(const Offsets& o, size_t L) { return o.line_v[L] + o.seg_v[L / kSegment]; }

// p_c = ((o_c + D[c][0] (s_x x)) + D[c][1] (s_y y)) + D[c][2] (s_z z), every operation rounded on its own.
__device__ __forceinline__ void place(const MeshPlacement& P, int u0, int u1, int u2, double* out) {
  const double tx = __dmul_rn(P.s[0], __dmul_rn((double)u2, 0.5)), ty = __dmul_rn(P.s[1], __dmul_rn((double)u1, 0.5)),
               tz = __dmul_rn(P.s[2], __dmul_rn((double)u0, 0.5));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double p = __dadd_rn(__dadd_rn(__dadd_rn(P.o[c], __dmul_rn(P.d[c * 3], tx)), __dmul_rn(P.d[c * 3 + 1], ty)),
                               __dmul_rn(P.d[c * 3 + 2], tz));
    out[c] = (P.ras && c < 2) ? -p : p;
  }
}

__device__ __forceinline__ u64 pick4(int l, u64 a, u64 b, u64 c, u64 d) { return l == 0 ? a : (l == 1 ? b : (l == 2 ? c : d)); }

__global__ void __launch_bounds__(kThreads) mesh_emit_kernel(const uint8_t* __restrict__ mask, MeshGeo g,
                                                            const int32_t* __restrict__ t_off,
                                                            const uint8_t* __restrict__ t_codes, int n_codes, size_t lines,
                                                            Offsets off, MeshPlacement P, int32_t* __restrict__ index2,
                                                            double* __restrict__ verts, int32_t* __restrict__ tris) {
  __shared__ int32_t s_off[kMeshConfigs + 1];
  __shared__ uint8_t s_codes[kMeshConfigs * kMeshMaxTriangles * 3];
  for (int i = threadIdx.x; i <= kMeshConfigs; i += blockDim.x) s_off[i] = t_off[i];
  for (int i = threadIdx.x; i < n_codes; i += blockDim.x) s_codes[i] = t_codes[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int n1p = g.n1 + 1;
  for (size_t L = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; L < lines; L += warps) {
    const int a = (int)(L / n1p), b = (int)(L % n1p);
    const int q0 = a - 1, q1 = b - 1;
    // vertex offsets of the lines (a + d0, b + d1) at the chunk start; a line past the grid has no vertices
    u64 vb0 = line_vertex_offset(off, L);
    u64 vb1 = b + 1 <= g.n1 ? line_vertex_offset(off, L + 1) : 0;
    u64 vb2 = a + 1 <= g.n0 ? line_vertex_offset(off, L + n1p) : 0;
    u64 vb3 = a + 1 <= g.n0 && b + 1 <= g.n1 ? line_vertex_offset(off, L + n1p + 1) : 0;
    u64 tb = off.line_t[L] + off.seg_t[L / kSegment];
    for (int x0 = -1; x0 < g.n2; x0 += 32) {
      const int x = x0 + lane;
      // row pairs (q0 + i, q1 + j), i, j in 0..2 but not both 2
      const unsigned r00 = member_pair(mask, g, q0, q1, x, lane), r01 = member_pair(mask, g, q0, q1 + 1, x, lane),
                     r02 = member_pair(mask, g, q0, q1 + 2, x, lane), r10 = member_pair(mask, g, q0 + 1, q1, x, lane),
                     r11 = member_pair(mask, g, q0 + 1, q1 + 1, x, lane),
                     r12 = member_pair(mask, g, q0 + 1, q1 + 2, x, lane), r20 = member_pair(mask, g, q0 + 2, q1, x, lane),
                     r21 = member_pair(mask, g, q0 + 2, q1 + 1, x, lane);
      const unsigned all = r00 | r01 | r02 | r10 | r11 | r12 | r20 | r21, none = r00 & r01 & r02 & r10 & r11 & r12 & r20 & r21;
      if (__all_sync(kFull, all == 0u || none == 3u)) continue;
      // line l = 2 d0 + d1: vertex bits at x, bit 0 at x + 1, vertices before x in the chunk, vertices in the chunk
      const unsigned vb[4] = {vertex_bits(r00, r10, r01), vertex_bits(r01, r11, r02), vertex_bits(r10, r20, r11),
                              vertex_bits(r11, r21, r12)};
      const unsigned nx[4] = {((r00 ^ r10) >> 1) & 1u, ((r01 ^ r11) >> 1) & 1u, ((r10 ^ r20) >> 1) & 1u,
                              ((r11 ^ r21) >> 1) & 1u};
      unsigned ex[4], tot[4];
#pragma unroll
      for (int l = 0; l < 4; ++l) {
        const unsigned b0 = __ballot_sync(kFull, vb[l] & 1u), b1 = __ballot_sync(kFull, vb[l] & 2u),
                       b2 = __ballot_sync(kFull, vb[l] & 4u);
        ex[l] = __popc(b0 & below) + __popc(b1 & below) + __popc(b2 & below);
        tot[l] = __popc(b0) + __popc(b1) + __popc(b2);
      }
      // the line's own vertices
      if (vb[0]) {
        u64 id = vb0 + ex[0];
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          if (!(vb[0] & (1u << m))) continue;
          const int u0 = 2 * q0 + (m == 0), u1 = 2 * q1 + (m == 1), u2 = 2 * x + (m == 2);
          index2[id * 3] = u0;
          index2[id * 3 + 1] = u1;
          index2[id * 3 + 2] = u2;
          double p[3];
          place(P, u0, u1, u2, p);
          verts[id * 3] = p[0];
          verts[id * 3 + 1] = p[1];
          verts[id * 3 + 2] = p[2];
          ++id;
        }
      }
      // the cube's triangles
      const unsigned c = cube_config(r00, r01, r10, r11);
      const int first = s_off[c], nt = s_off[c + 1] - first;
      int inc = nt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(kFull, inc, o);
        if (lane >= o) inc += y;
      }
      const int chunk_t = __shfl_sync(kFull, inc, 31);
      u64 tid = tb + (unsigned)(inc - nt);
      for (int t = 0; t < nt; ++t, ++tid) {
        int32_t ids[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const unsigned code = s_codes[(first + t) * 3 + k];
          const int corner = (int)(code >> 2), m = (int)(code & 3u), l = corner >> 1, d2 = corner & 1;
          const unsigned bits = l == 0 ? vb[0] : (l == 1 ? vb[1] : (l == 2 ? vb[2] : vb[3]));
          const unsigned next0 = l == 0 ? nx[0] : (l == 1 ? nx[1] : (l == 2 ? nx[2] : nx[3]));
          const unsigned e = l == 0 ? ex[0] : (l == 1 ? ex[1] : (l == 2 ? ex[2] : ex[3]));
          // vertices before (x + d2) on line l, then the rank of m among the point's bits (an edge with d2 = 1 has m < 2)
          const unsigned before = e + (d2 ? __popc(bits) : 0u);
          const unsigned rank = m == 0 ? 0u : (m == 1 ? (d2 ? next0 : (bits & 1u)) : __popc(bits & 3u));
          ids[k] = (int32_t)(pick4(l, vb0, vb1, vb2, vb3) + before + rank);
        }
        tris[tid * 3] = ids[0];
        tris[tid * 3 + 1] = P.reverse ? ids[2] : ids[1];
        tris[tid * 3 + 2] = P.reverse ? ids[1] : ids[2];
      }
      vb0 += tot[0];
      vb1 += tot[1];
      vb2 += tot[2];
      vb3 += tot[3];
      tb += (unsigned)chunk_t;
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
#define MC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

template <typename K>
int warp_grid(K kernel, size_t lines, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (lines * 32 + kThreads - 1) / kThreads;
  return (int)std::max<size_t>(std::min((size_t)per_sm * num_sms, need), 1);
}

// The work area: table offsets | table codes | per-line V | per-line T | segment V | segment T.
struct Layout {
  int32_t* off;
  uint8_t* codes;
  u64 *cnt_v, *cnt_t, *seg_v, *seg_t;
  size_t lines;
  int segs, n_codes;
};

int layout(MeshWork& w, int n0, int n1, const MeshTable& tab, cudaStream_t st, Layout& o) {
  o.lines = (size_t)(n0 + 1) * (n1 + 1);
  o.segs = (int)((o.lines + kSegment - 1) / kSegment);
  o.n_codes = tab.off[kMeshConfigs] * 3;
  const size_t o_codes = align256((kMeshConfigs + 1) * sizeof(int32_t)), o_v = o_codes + align256(o.n_codes);
  const size_t o_t = o_v + align256(o.lines * sizeof(u64)), o_sv = o_t + align256(o.lines * sizeof(u64));
  const size_t o_st = o_sv + align256((o.segs + 1) * sizeof(u64)), bytes = o_st + (o.segs + 1) * sizeof(u64);
  MC((cudaError_t)w.reserve(bytes));
  char* base = static_cast<char*>(w.d);
  o.off = reinterpret_cast<int32_t*>(base);
  o.codes = reinterpret_cast<uint8_t*>(base + o_codes);
  o.cnt_v = reinterpret_cast<u64*>(base + o_v);
  o.cnt_t = reinterpret_cast<u64*>(base + o_t);
  o.seg_v = reinterpret_cast<u64*>(base + o_sv);
  o.seg_t = reinterpret_cast<u64*>(base + o_st);
  MC(cudaMemcpyAsync(o.off, tab.off, (kMeshConfigs + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (o.n_codes) MC(cudaMemcpyAsync(o.codes, tab.codes, o.n_codes, cudaMemcpyHostToDevice, st));
  return 0;
}

// Count pass and scan; the totals to the host.  Synchronises `st`.
int count_and_scan(const Layout& o, const uint8_t* d_mask, const MeshGeo& g, int num_sms, cudaStream_t st,
                   int64_t* launches, int64_t* n_vertices, int64_t* n_triangles) {
  mesh_count_kernel<<<warp_grid(mesh_count_kernel, o.lines, num_sms), kThreads, 0, st>>>(d_mask, g, o.off, o.lines, o.cnt_v,
                                                                                         o.cnt_t);
  MC(cudaGetLastError());
  mesh_scan_kernel<<<o.segs, kScanThreads, 0, st>>>(o.cnt_v, o.cnt_t, o.lines, o.seg_v, o.seg_t);
  MC(cudaGetLastError());
  mesh_scan_top_kernel<<<1, kScanThreads, 0, st>>>(o.seg_v, o.seg_t, o.segs);
  MC(cudaGetLastError());
  *launches += 3;
  u64 tot[2];
  MC(cudaMemcpyAsync(&tot[0], o.seg_v + o.segs, sizeof(u64), cudaMemcpyDeviceToHost, st));
  MC(cudaMemcpyAsync(&tot[1], o.seg_t + o.segs, sizeof(u64), cudaMemcpyDeviceToHost, st));
  MC(cudaStreamSynchronize(st));
  *n_vertices = (int64_t)tot[0];
  *n_triangles = (int64_t)tot[1];
  return 0;
}

}  // namespace

int MeshWork::reserve(size_t need) {
  if (need <= bytes) return 0;
  if (d) cudaFree(d);
  d = nullptr;
  bytes = 0;
  MC(cudaMalloc(&d, need));
  bytes = need;
  return 0;
}

void MeshWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  bytes = 0;
}

int mesh_counts(MeshWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const MeshTable& tab, int64_t* n_vertices,
                int64_t* n_triangles, int num_sms, cudaStream_t st, int64_t* launches) {
  Layout o;
  MC((cudaError_t)layout(w, n0, n1, tab, st, o));
  return count_and_scan(o, d_mask, MeshGeo{n0, n1, n2, row}, num_sms, st, launches, n_vertices, n_triangles);
}

int mesh_emit(MeshWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const MeshTable& tab,
              const MeshPlacement& placement, int64_t n_vertices, int64_t n_triangles, int32_t* d_index2,
              double* d_vertices, int32_t* d_triangles, int num_sms, cudaStream_t st, int64_t* launches) {
  Layout o;
  MC((cudaError_t)layout(w, n0, n1, tab, st, o));
  const MeshGeo g{n0, n1, n2, row};
  int64_t nv = 0, nt = 0;
  MC((cudaError_t)count_and_scan(o, d_mask, g, num_sms, st, launches, &nv, &nt));
  if (nv != n_vertices || nt != n_triangles) return -2;
  if (!nv && !nt) return 0;
  const Offsets off{o.cnt_v, o.cnt_t, o.seg_v, o.seg_t};
  mesh_emit_kernel<<<warp_grid(mesh_emit_kernel, o.lines, num_sms), kThreads, 0, st>>>(
      d_mask, g, o.off, o.codes, o.n_codes, o.lines, off, placement, d_index2, d_vertices, d_triangles);
  MC(cudaGetLastError());
  ++*launches;
  MC(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace lm
