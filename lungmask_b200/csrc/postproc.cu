// Post-processing on device: utils.postprocessing (utils.py:272-358), utils.reshape_mask (utils.py:114-129)
// and the fusion glue of LMInferer.apply (mask.py:228-230).  Integer work, bit-exact with the reference
// (oracle/restate.py is the CPU statement of the same algorithm).
//
//  Q1  26-connected components of equal label value: union-find over the voxel grid (roots = minimum linear
//      index, so ranking the roots reproduces skimage's raster-order ids)               utils.py:293
//  Q2  per region: area, label value, bounding box                                      utils.py:298
//  Q3  ascending (area, id) order by a bitonic sort of 64-bit keys + the per-label "record" pass restated
//      order-free (a region sets a record iff it has the lowest id among the regions of its value AND area;
//      the final record of a value is its largest area), all on device                   utils.py:299-308
//  Q4  the order-dependent merge loop runs in ONE persistent CTA on the device: per candidate region it
//      scans the region's (growing) bounding box, histograms the ids of the 6-connected ring voxels, picks
//      the max-count / lowest-id neighbour and updates area / record / redirect tables   utils.py:310-339
//  Q5  region -> label map, spare labels zeroed                                         utils.py:341-342
//  Q6  per label: largest 26-connected component, then holes (background not 6-connected to the border,
//      or 2-D 4-connected background components < 64 px for single-slice volumes) filled, painted in
//      ascending label order                                                            utils.py:344-358
//
// Round 2: the host is out of the loop.  The region count R, the sort, the records, the per-label boxes and the
// "is this label present" decisions stay in device memory; kernels read them there (grids are sized for the volume,
// loops for the device-side bounds).  With a known label bound the whole post-processing is enqueued without a single
// host synchronisation (one when the bound is unknown); the region tables have a capacity and the device raises a
// flag when R exceeds it (postprocess_finish -> the caller grows the tables and runs again).
#include <algorithm>
#include <atomic>
#include <vector>
#include <string.h>
#include <cooperative_groups.h>
#include "postproc.cuh"

namespace cg = cooperative_groups;

namespace lm {
namespace {

constexpr uint32_t NONE = 0xFFFFFFFFu;

struct Box { int z0, z1, y0, y1, x0, x1; };  // half-open
struct Dim { int S, H, W; };
// A box known on the host (dyn == nullptr) or the extent [z0,z1,y0,y1,x0,x1) in device memory grown by one voxel and
// clipped (the analysis box of the hole filling); `gate` (optional) points to a device flag: 0 = the kernel has nothing to do.
struct BoxSrc { Box fixed; const int* dyn; const uint32_t* gate; };

__device__ __forceinline__ bool resolve_box(const BoxSrc& s, const Dim& d, Box& b) {
  if (s.gate && *s.gate == 0u) return false;
  if (!s.dyn) { b = s.fixed; return true; }
  if (s.dyn[1] < 0) return false;  // empty extent
  b.z0 = max(s.dyn[0] - 1, 0); b.z1 = min(s.dyn[1] + 1, d.S);
  b.y0 = max(s.dyn[2] - 1, 0); b.y1 = min(s.dyn[3] + 1, d.H);
  b.x0 = max(s.dyn[4] - 1, 0); b.x1 = min(s.dyn[5] + 1, d.W);
  return true;
}

__device__ __forceinline__ uint32_t uf_find(uint32_t* parent, uint32_t i) {
  uint32_t p = parent[i];
  while (p != i) {
    const uint32_t g = parent[p];
    if (g != p) parent[i] = g;  // path halving (benign race: always an ancestor)
    i = p;
    p = g;
  }
  return i;
}
__device__ __forceinline__ void uf_union(uint32_t* parent, uint32_t a, uint32_t b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const uint32_t t = a; a = b; b = t; }
    const uint32_t old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}

__device__ __forceinline__ size_t box_volume(const Box& b) {
  return (size_t)(b.z1 - b.z0) * (b.y1 - b.y0) * (b.x1 - b.x0);
}
// t-th voxel of the box -> (z,y,x) and linear index in the full volume.  Volumes hold fewer than 2^32 voxels
// (postprocess_device refuses more), so the index arithmetic is 32-bit: two unsigned divisions instead of four 64-bit
// ones - the r02 launch list showed the labelling kernels instruction-bound on exactly that.
__device__ __forceinline__ uint32_t box_voxel(const Box& b, const Dim& d, size_t t, int& z, int& y, int& x) {
  const uint32_t bw = (uint32_t)(b.x1 - b.x0), bh = (uint32_t)(b.y1 - b.y0), tt = (uint32_t)t;
  const uint32_t r = tt / bw;
  x = b.x0 + (int)(tt - r * bw);
  const uint32_t zz = r / bh;
  y = b.y0 + (int)(r - zz * bh);
  z = b.z0 + (int)zz;
  return ((uint32_t)z * (uint32_t)d.H + (uint32_t)y) * (uint32_t)d.W + (uint32_t)x;
}
// linear index -> (z,y,x), 32-bit
__device__ __forceinline__ void voxel_zyx(const Dim& d, uint32_t i, int& z, int& y, int& x) {
  const uint32_t r = i / (uint32_t)d.W;
  x = (int)(i - r * (uint32_t)d.W);
  const uint32_t zz = r / (uint32_t)d.H;
  y = (int)(r - zz * (uint32_t)d.H);
  z = (int)zz;
}

// Union-find initialisation.  Consecutive threads hold consecutive voxels of a row, so the x-runs of equal label are
// linked here without atomics: every voxel points at the first voxel of its run WITHIN the warp's 32-voxel segment
// (a run start is the smallest index of the run: the min-index-root invariant holds); the merge kernel joins the
// segments (lane 0 only).  All lanes run the same number of iterations (the ballot needs them).
__global__ void ccl_init_kernel(const uint8_t* __restrict__ vals, uint32_t* __restrict__ parent, Dim d, BoxSrc bs) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  const unsigned lane = threadIdx.x & 31u;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t0 = blockIdx.x * (size_t)blockDim.x + (threadIdx.x - lane); t0 < n; t0 += stride) {
    const size_t t = t0 + lane;
    uint32_t i = 0;
    uint8_t v = 0;
    bool left = false;
    if (t < n) {
      int z, y, x;
      i = box_voxel(b, d, t, z, y, x);
      v = vals[i];
      left = v && lane > 0 && x > b.x0 && vals[i - 1] == v;
    }
    const unsigned m = __ballot_sync(0xffffffffu, left);
    if (t < n) {
      uint32_t p = NONE;
      if (v) {
        const unsigned stops = ~m & (0xffffffffu >> (31u - lane));  // lanes <= this one that start a run (lane 0 always does)
        const unsigned start = 31u - (unsigned)__clz(stops);
        p = i - (lane - start);
      }
      parent[i] = p;
    }
  }
}

// CONN: 26 (3-D full), 6 (3-D faces), 4 (2-D faces within a slice). Only neighbours inside the box count.
// The x-runs are already linked inside every 32-voxel segment (ccl_init_kernel); here lane 0 joins the segments and each
// voxel is united with its backward neighbours in the four rows (y-1,z), (y-1,z-1), (y,z-1), (y+1,z-1).
// rule != 0 (CONN == 26; the default): per backward row with a = (x-1), b = (x), c = (x+1) of that row,
//     b same label            -> unite with b, unless the left voxel carries the label too (it is united with b's row
//                                through its own c or b, and b's row neighbours are linked by their own left links)
//     b differs               -> unite with c if it matches; with a only if the left voxel does not carry the label
// which performs no union at all inside homogeneous regions.  Same partition and same minimum-index roots as probing
// all 13 backward neighbours (rule == 0): proof by induction along the row in DESIGN.md section 4.3; the CPU enumeration
// is tests/test_ccl_neighbour_rule.py, the GPU comparison tests/test_gpu_stages.py::test_ccl_rules_agree.
template <int CONN>
__global__ void ccl_merge_kernel(const uint8_t* __restrict__ vals, uint32_t* __restrict__ parent, Dim d, BoxSrc bs, int rule) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  const size_t HW = (size_t)d.H * d.W;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    const uint8_t v = vals[i];
    if (!v) continue;
    const bool left = x > b.x0 && vals[i - 1] == v;
    if (left && (threadIdx.x & 31) == 0) uf_union(parent, i, i - 1);  // the run continues across a 32-voxel segment
    if (CONN == 26) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int dy = (r == 3) ? 1 : (r == 2 ? 0 : -1), dz = (r == 0) ? 0 : -1;
        const int yy = y + dy, zz = z + dz;
        if (zz < b.z0 || yy < b.y0 || yy >= b.y1) continue;
        const uint32_t j = (uint32_t)((size_t)zz * HW + (size_t)yy * d.W + x);
        const bool sb = vals[j] == v;
        const bool sa = x > b.x0 && vals[j - 1] == v;
        const bool sc = x + 1 < b.x1 && vals[j + 1] == v;
        if (rule) {
          if (sb) { if (!left) uf_union(parent, i, j); continue; }
          if (sa && !left) uf_union(parent, i, j - 1);
          if (sc) uf_union(parent, i, j + 1);
        } else {
          if (sa) uf_union(parent, i, j - 1);
          if (sb) uf_union(parent, i, j);
          if (sc) uf_union(parent, i, j + 1);
        }
      }
    } else {
      // faces only: the upper / previous-slice neighbour needs no union when the left voxel and ITS upper neighbour
      // carry the label as well (left link + the neighbour's own left link close the square)
      if (y > b.y0 && vals[i - d.W] == v && !(left && vals[i - d.W - 1] == v)) uf_union(parent, i, i - d.W);
      if (CONN == 6 && z > b.z0 && vals[i - HW] == v && !(left && vals[i - HW - 1] == v)) uf_union(parent, i, (uint32_t)(i - HW));
    }
  }
}

// Joins slab-wise labellings (multi-GPU slice sharding, shard.cu): every slab [z_lo, z_hi) was labelled on its own
// with neighbours outside the slab ignored; here the voxels of each slab's FIRST slice are united with their nine
// backward neighbours in the previous slab's last slice.  Roots stay minimum linear indices, so the union of slab
// labellings plus these links is exactly the whole-volume labelling.  bounds: the first slices of slabs 1..n-1.
struct SlabBounds { int n; int z[16]; };
__global__ void ccl_join_slabs_kernel(const uint8_t* __restrict__ vals, uint32_t* __restrict__ parent, Dim d, SlabBounds sb) {
  const size_t HW = (size_t)d.H * d.W;
  const size_t total = (size_t)sb.n * HW;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const uint32_t bi = (uint32_t)t / (uint32_t)HW, r = (uint32_t)t - bi * (uint32_t)HW;
    const int z = sb.z[bi];
    const int y = (int)(r / (uint32_t)d.W), x = (int)(r - (uint32_t)y * (uint32_t)d.W);
    const uint32_t i = (uint32_t)((size_t)z * HW + r);
    const uint8_t v = vals[i];
    if (!v || z == 0) continue;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int yy = y + dy, xx = x + dx;
        if (yy < 0 || yy >= d.H || xx < 0 || xx >= d.W) continue;
        const uint32_t j = (uint32_t)((size_t)(z - 1) * HW + (size_t)yy * d.W + xx);
        if (vals[j] == v) uf_union(parent, i, j);
      }
  }
}

// Read-only walk: while flattening, a thread may only write its OWN slot; a path-halving write from another
// walker could overwrite an already flattened slot with a stale non-root ancestor.
__device__ __forceinline__ uint32_t uf_find_ro(const uint32_t* parent, uint32_t i) {
  uint32_t p = parent[i];
  while (p != i) { i = p; p = parent[i]; }
  return i;
}
__global__ void ccl_flatten_kernel(uint32_t* __restrict__ parent, Dim d, BoxSrc bs) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    if (parent[i] != NONE) parent[i] = uf_find_ro(parent, i);
  }
}

// ---- canonical ids: rank of each root in raster order (three-pass scan) -------------------------------
constexpr int SCAN_BLOCK = 1024, SCAN_ITEMS = 4;  // 4096 voxels per block
__global__ void __launch_bounds__(SCAN_BLOCK) roots_count_kernel(const uint32_t* __restrict__ parent, size_t n,
                                                                 uint32_t* __restrict__ block_counts) {
  __shared__ uint32_t ws[32];
  const size_t base = (size_t)blockIdx.x * SCAN_BLOCK * SCAN_ITEMS;
  uint32_t c = 0;
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    const size_t i = base + (size_t)k * SCAN_BLOCK + threadIdx.x;
    if (i < n && parent[i] == (uint32_t)i) ++c;
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x < 32) {
    c = ws[threadIdx.x];
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
  }
}
__global__ void __launch_bounds__(1024) scan_blocks_kernel(uint32_t* __restrict__ block_counts, int nb,
                                                           uint32_t* __restrict__ total) {
  __shared__ uint32_t ws[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t v = i < nb ? block_counts[i] : 0;
    uint32_t s = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, s, o); if ((threadIdx.x & 31) >= o) s += t; }
    if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = ws[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += t; }
      ws[threadIdx.x] = w;
    }
    __syncthreads();
    const uint32_t warp_off = (threadIdx.x >> 5) ? ws[(threadIdx.x >> 5) - 1] : 0;
    const uint32_t excl = carry + warp_off + s - v;
    if (i < nb) block_counts[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
// rid[root] = rank+1 ; serial within a block over its 4096 voxels in raster order (warp-scan per 1024 chunk)
__global__ void __launch_bounds__(SCAN_BLOCK) roots_assign_kernel(const uint32_t* __restrict__ parent, size_t n,
                                                                  const uint32_t* __restrict__ block_offsets,
                                                                  uint32_t* __restrict__ rid) {
  __shared__ uint32_t ws[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = block_offsets[blockIdx.x];
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * SCAN_BLOCK * SCAN_ITEMS;
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    const size_t i = base + (size_t)k * SCAN_BLOCK + threadIdx.x;
    const uint32_t f = (i < n && parent[i] == (uint32_t)i) ? 1u : 0u;
    uint32_t s = f;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, s, o); if ((threadIdx.x & 31) >= o) s += t; }
    if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = ws[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += t; }
      ws[threadIdx.x] = w;
    }
    __syncthreads();
    const uint32_t incl = carry + ((threadIdx.x >> 5) ? ws[(threadIdx.x >> 5) - 1] : 0) + s;
    if (f) rid[i] = incl;  // 1-based id
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
}

// ---- small device tables (PostScratch::small, 32 KB) ----------------------------------------------------------
// words: [0] largest R since the host last looked  [1] region-table overflow flag (sticky until then)
//        [2] first present label value  [3] "label active" gate of the Q6 loop  [4] R of this run
//        [8..264) present[256]  [512..768) record[256] (origlabels_maxsub)
// bytes: [4096..4352) spare_value[256]   [8192..10240) best root per label value (u64[256])
//        [16384..16408) extent of the label being finalised (int[6])   [16640..) spare label values (int32[16])
constexpr int W_MAXR = 0, W_OVERFLOW = 1, W_FIRST = 2, W_GATE = 3, W_R = 4, W_PRESENT = 8, W_RECORD = 512;
constexpr int B_SPARE_VALUE = 4096, B_BEST = 8192, B_BBOX1 = 16384, B_SPARE_LIST = 16640;
constexpr int MAX_SPARE = 16;

struct SpareArgs { int n; int v[MAX_SPARE]; const int32_t* d_extra; int n_extra; };

// spare tables + record / present / best reset (one block)
__global__ void post_setup_kernel(uint32_t* small, SpareArgs sp, int clear_sticky) {
  uint8_t* spare_value = reinterpret_cast<uint8_t*>(small) + B_SPARE_VALUE;
  int32_t* spare_list = reinterpret_cast<int32_t*>(reinterpret_cast<uint8_t*>(small) + B_SPARE_LIST);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(small) + B_BEST);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    spare_value[i] = 0;
    small[W_PRESENT + i] = 0;
    small[W_RECORD + i] = 0;
    best[i] = 0ull;
  }
  if (threadIdx.x == 0) {
    small[W_GATE] = 0; small[W_FIRST] = 0;
    if (clear_sticky) { small[W_OVERFLOW] = 0; small[W_MAXR] = 0; }
  }
  __syncthreads();
  const int total = sp.n + sp.n_extra;
  for (int i = threadIdx.x; i < MAX_SPARE; i += blockDim.x) {
    int v = -1;
    if (i < sp.n) v = sp.v[i];
    else if (i < total) v = sp.d_extra[i - sp.n];
    spare_list[i] = v;
    if (v >= 0 && v < 256) spare_value[v] = 1;
  }
}

// region tables for ids 0..min(R, cap): zero / identity, spare_id[i] = "the ID i equals a spare entry" (utils.py:322)
__global__ void region_init_kernel(uint32_t* small, uint32_t cap, uint32_t* __restrict__ area,
                                   uint32_t* __restrict__ count, uint8_t* __restrict__ value, int* __restrict__ bbox,
                                   uint32_t* __restrict__ cur, uint8_t* __restrict__ to_label, uint8_t* __restrict__ spare_id) {
  const uint32_t R = small[W_R];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    atomicMax(&small[W_MAXR], R);
    if (R > cap) small[W_OVERFLOW] = 1;
  }
  const uint32_t top = R < cap ? R : cap;
  const int32_t* spare_list = reinterpret_cast<const int32_t*>(reinterpret_cast<const uint8_t*>(small) + B_SPARE_LIST);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= top; i += gridDim.x * blockDim.x) {
    area[i] = 0; count[i] = 0; value[i] = 0; cur[i] = i; to_label[i] = 0;
    int* b = bbox + 6 * (size_t)i;
    b[0] = b[2] = b[4] = 1 << 30;
    b[1] = b[3] = b[5] = -1;
    uint8_t s = 0;
#pragma unroll
    for (int k = 0; k < MAX_SPARE; ++k) s |= (spare_list[k] >= 0 && (uint32_t)spare_list[k] == i) ? 1 : 0;
    spare_id[i] = s;
  }
}

// rid for every voxel (0 = background) + region statistics
__global__ void region_stats_kernel(const uint8_t* __restrict__ vals, const uint32_t* __restrict__ parent,
                                    uint32_t* __restrict__ rid, Dim d, uint32_t cap, uint32_t* __restrict__ area,
                                    uint8_t* __restrict__ value, int* __restrict__ bbox) {
  const size_t n = (size_t)d.S * d.H * d.W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t p = parent[i];
    if (p == NONE) { rid[i] = 0; continue; }
    const uint32_t id = rid[p];  // roots were assigned by roots_assign_kernel; non-roots never alias a root slot
    if (p != (uint32_t)i) rid[i] = id;
    if (id > cap) continue;      // table overflow: flagged by region_init_kernel, the caller runs again with larger tables
    if (p == (uint32_t)i) value[id] = vals[i];
    // warp-aggregated area count
    const unsigned peers = __match_any_sync(__activemask(), id);
    if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&area[id], (uint32_t)__popc(peers));
    int x, y, z;
    voxel_zyx(d, (uint32_t)i, z, y, x);
    int* bb = bbox + 6 * (size_t)id;
    if (z < bb[0]) atomicMin(&bb[0], z);
    if (z + 1 > bb[1]) atomicMax(&bb[1], z + 1);
    if (y < bb[2]) atomicMin(&bb[2], y);
    if (y + 1 > bb[3]) atomicMax(&bb[3], y + 1);
    if (x < bb[4]) atomicMin(&bb[4], x);
    if (x + 1 > bb[5]) atomicMax(&bb[5], x + 1);
  }
}

// ---- Q2/Q3 on device ---------------------------------------------------------------------------------------
// order[k] = id of the k-th region in ascending (area, id) order (Python's stable sort of the id-ordered list,
// utils.py:299-300): bitonic sort of the keys area << 32 | id by ONE CTA - in shared memory up to 4096 regions, in
// global memory above (R is a device-side value; a clean label map has tens of regions, a speckled one thousands).
constexpr int SORT_SMEM = 4096;
__device__ __forceinline__ void bitonic_pass(unsigned long long* keys, uint32_t npad, uint32_t k, uint32_t j) {
  for (uint32_t i = threadIdx.x; i < npad; i += blockDim.x) {
    const uint32_t l = i ^ j;
    if (l > i) {
      const unsigned long long a = keys[i], b = keys[l];
      const bool up = (i & k) == 0;
      if ((a > b) == up) { keys[i] = b; keys[l] = a; }
    }
  }
}
__global__ void __launch_bounds__(1024, 1) region_sort_kernel(const uint32_t* __restrict__ small, uint32_t cap,
                                                              const uint32_t* __restrict__ area,
                                                              unsigned long long* __restrict__ gkeys,
                                                              uint32_t* __restrict__ order) {
  __shared__ unsigned long long skeys[SORT_SMEM];
  const uint32_t R = small[W_R] < cap ? small[W_R] : cap;
  if (R == 0) return;
  uint32_t npad = 2;
  while (npad < R) npad <<= 1;
  unsigned long long* keys = npad <= SORT_SMEM ? skeys : gkeys;
  for (uint32_t i = threadIdx.x; i < npad; i += blockDim.x)
    keys[i] = i < R ? (((unsigned long long)area[i + 1] << 32) | (unsigned long long)(i + 1)) : ~0ull;
  __syncthreads();
  for (uint32_t k = 2; k <= npad; k <<= 1)
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      bitonic_pass(keys, npad, k, j);
      __syncthreads();
    }
  for (uint32_t i = threadIdx.x; i < R; i += blockDim.x) order[i] = (uint32_t)(keys[i] & 0xFFFFFFFFull);
}

// Records (utils.py:303-308) without walking the sorted list: going through the regions in ascending (area, id) order,
// a region sets a new record for its label value v iff its area is strictly larger than every earlier region of value
// v, i.e. iff no region of value v with the SAME area has a lower id; the record left at the end is the largest area of
// value v.  (area, v) -> lowest id through an open-addressing table.
__device__ __forceinline__ uint32_t hash40(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}
__global__ void record_insert_kernel(uint32_t* __restrict__ small, uint32_t cap, const uint32_t* __restrict__ area,
                                     const uint8_t* __restrict__ value, unsigned long long* __restrict__ hkeys,
                                     uint32_t* __restrict__ hmin, uint32_t hmask, uint32_t* __restrict__ hslot) {
  __shared__ uint32_t srec[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) srec[i] = 0;
  __syncthreads();
  const uint32_t R = small[W_R] < cap ? small[W_R] : cap;
  for (uint32_t id = 1 + blockIdx.x * blockDim.x + threadIdx.x; id <= R; id += gridDim.x * blockDim.x) {
    const uint32_t a = area[id];
    const uint8_t v = value[id];
    atomicMax(&srec[v], a);
    const unsigned long long key = ((unsigned long long)a << 8) | v;
    uint32_t s = hash40(key) & hmask;
    while (true) {
      const unsigned long long prev = atomicCAS(&hkeys[s], ~0ull, key);
      if (prev == ~0ull || prev == key) break;
      s = (s + 1) & hmask;
    }
    atomicMin(&hmin[s], id);
    hslot[id] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (srec[i]) atomicMax(&small[W_RECORD + i], srec[i]);
}
__global__ void record_lookup_kernel(const uint32_t* __restrict__ small, uint32_t cap, const uint8_t* __restrict__ value,
                                     const uint32_t* __restrict__ hmin, const uint32_t* __restrict__ hslot,
                                     uint8_t* __restrict__ to_label) {
  const uint32_t R = small[W_R] < cap ? small[W_R] : cap;
  for (uint32_t id = 1 + blockIdx.x * blockDim.x + threadIdx.x; id <= R; id += gridDim.x * blockDim.x)
    to_label[id] = (hmin[hslot[id]] == id) ? value[id] : 0;
}

// ---- Q4: the sequential merge loop, one persistent CTA ---------------------------------------------------
__device__ __forceinline__ uint32_t cur_find(uint32_t* cur, uint32_t id) {
  uint32_t p = cur[id];
  while (p != id) {
    const uint32_t g = cur[p];
    if (g != p) cur[id] = g;
    id = p;
    p = g;
  }
  return id;
}

struct MergeArgs {
  const uint32_t* rid;     // [Nv] original region id per voxel
  uint32_t* cur;           // [R+1] redirect (regionmask[regionmask == id] = mapto)
  uint32_t* area;          // [R+1] cached areas (mutated, utils.py:339)
  const uint8_t* value;    // [R+1] label value of each region (max_intensity)
  int* bbox;               // [R+1][6] current extent
  uint32_t* record;        // [256] origlabels_maxsub
  const uint32_t* order;   // [R] region ids in ascending (area, id) order
  uint32_t* count;         // [R+1] scratch, zero on entry and exit
  uint32_t* touched;       // [R+1] scratch
  const uint8_t* spare_value;  // [256] 1 where the label VALUE is spare            (utils.py:313: v in spare)
  const uint8_t* spare_id;     // [R+1] 1 where the region ID equals a spare entry  (utils.py:322: n not in spare)
  const uint32_t* d_R;     // device-side region count
  uint32_t cap;            // table capacity (ids above it do not exist in the tables)
  int skip_below;
  Dim d;
};

// The sequential loop over the order positions [k0, k1): what utils.py:310-339 does, one candidate at a time, by ONE CTA
// (any block size).  Used for small region counts and for the rare candidate whose neighbour set does not fit the
// per-CTA table of the multi-CTA kernel below.
__device__ void merge_serial_range(const MergeArgs& a, uint32_t k0, uint32_t k1) {
  __shared__ uint32_t s_first;
  __shared__ Box s_box;
  __shared__ uint32_t s_ntouched;
  __shared__ unsigned long long s_best;
  const int tid = threadIdx.x;
  const Dim d = a.d;
  const size_t HW = (size_t)d.H * d.W;
  uint32_t k = k0;
  while (k < k1) {
    // The tables only change when a candidate is processed, so the next candidate can be searched for
    // blockDim regions at a time; the first hit (in list order) is the one the sequential loop would take.
    if (tid == 0) s_first = NONE;
    __syncthreads();
    if (k + tid < k1) {
      const uint32_t rr = a.order[k + tid];
      const uint32_t ar = a.area[rr];
      const uint8_t v = a.value[rr];
      if ((ar < a.record[v] || a.spare_value[v]) && ar >= (uint32_t)a.skip_below) atomicMin(&s_first, k + (uint32_t)tid);
    }
    __syncthreads();
    const uint32_t kk = s_first;
    if (kk == NONE) { k += blockDim.x; __syncthreads(); continue; }
    const uint32_t r = a.order[kk];
    k = kk + 1;
    if (tid == 0) {
      const int* bb = a.bbox + 6 * (size_t)r;  // ring voxels lie within the extent grown by one
      s_box.z0 = max(bb[0] - 1, 0); s_box.z1 = min(bb[1] + 1, d.S);
      s_box.y0 = max(bb[2] - 1, 0); s_box.y1 = min(bb[3] + 1, d.H);
      s_box.x0 = max(bb[4] - 1, 0); s_box.x1 = min(bb[5] + 1, d.W);
      s_ntouched = 0;
      s_best = 0ull;
    }
    __syncthreads();
    const Box b = s_box;
    const size_t n = box_volume(b);
    for (size_t t = tid; t < n; t += blockDim.x) {
      int z, y, x;
      const uint32_t i = box_voxel(b, d, t, z, y, x);
      const uint32_t o = a.rid[i];
      if (o == 0 || o > a.cap) continue;  // n != 0 (ids beyond the tables exist only in an overflowed run, which is repeated)
      const uint32_t id = cur_find(a.cur, o);
      if (id == r) continue;  // n != r.label
      bool ring = false;  // binary_dilation(sub == r.label), 6-connected cross (utils.py:316)
      if (x > 0)       { const uint32_t q = a.rid[i - 1];        ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (x < d.W - 1) { const uint32_t q = a.rid[i + 1];        ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (y > 0)       { const uint32_t q = a.rid[i - d.W];      ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (y < d.H - 1) { const uint32_t q = a.rid[i + d.W];      ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (z > 0)       { const uint32_t q = a.rid[i - HW];       ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (z < d.S - 1) { const uint32_t q = a.rid[i + HW];       ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
      if (!ring) continue;
      if (atomicAdd(&a.count[id], 1u) == 0u) a.touched[atomicAdd(&s_ntouched, 1u)] = id;
    }
    __syncthreads();
    const uint32_t nt = s_ntouched;
    for (uint32_t t = tid; t < nt; t += blockDim.x) {
      const uint32_t id = a.touched[t];
      const uint32_t c = a.count[id];
      a.count[id] = 0;
      if (a.spare_id[id]) continue;
      // max count; strict '>' while scanning ids ascending  =>  lowest id wins ties
      atomicMax(&s_best, ((unsigned long long)c << 32) | (unsigned long long)(0xFFFFFFFFu - id));
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t mapto = r, moved = 0;
      if (s_best != 0ull) { mapto = 0xFFFFFFFFu - (uint32_t)(s_best & 0xFFFFFFFFull); moved = a.area[r]; }
      if (mapto != r) {
        a.cur[r] = mapto;
        int* bt = a.bbox + 6 * (size_t)mapto;
        const int* br = a.bbox + 6 * (size_t)r;
        bt[0] = min(bt[0], br[0]); bt[1] = max(bt[1], br[1]);
        bt[2] = min(bt[2], br[2]); bt[3] = max(bt[3], br[3]);
        bt[4] = min(bt[4], br[4]); bt[5] = max(bt[5], br[5]);
      }
      const uint8_t tv = a.value[mapto];
      if (a.area[mapto] == a.record[tv]) a.record[tv] += moved;
      a.area[mapto] += moved;
      __threadfence();
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024, 1) merge_loop_kernel(MergeArgs a) {
  const uint32_t R = *a.d_R < a.cap ? *a.d_R : a.cap;
  merge_serial_range(a, 0, R);
}

// ---- Q4 on many CTAs ---------------------------------------------------------------------------------------------
// The loop is sequential by definition (every merge changes the label map the next candidate sees), but candidates
// whose extents are not even adjacent cannot see each other's merges: a merge of region i into its neighbour changes
// (a) the ids of i's voxels, which only matter to a candidate j if they lie in j's ring - impossible when the boxes
// of i and j are separated by a voxel - and (b) the target's area / record, which are applied in order afterwards.
// So the kernel processes the order in BATCHES: the longest prefix of upcoming candidates whose extents are pairwise
// separated (and that is not interrupted by a region a record growth could turn into a candidate).
//   build (CTA 0)    classify a window of the order with the current tables, list the candidates in order, cut at the
//                    first one that touches an earlier one
//   decide (all)     one CTA per batch member: ring histogram in a shared-memory table, max count / lowest id -> target
//   apply (CTA 0)    the area / record arithmetic of utils.py:333-339 sequentially in order on shared-memory copies
//                    (tens of cycles per member), then cur / bbox / area / record written back in parallel; a merge that
//                    lifts a skipped (< skip_below) region inside the batch's span over the threshold truncates the batch
//                    there (that region becomes a candidate at its turn)
// two grid-wide synchronisations per batch (cooperative launch).  tests: the CPU emulation of exactly this schedule
// against the sequential loop (tests/test_merge_batches.py) and the bit-exact post-processing tests with either kernel.
constexpr int MC_THREADS = 512;
constexpr int MC_BMAX = 256;      // members per batch
constexpr int MC_WINDOW = 2048;   // order positions classified per build step
constexpr int MC_HASH = 1024;     // neighbour ids per candidate in the per-CTA table (more: the serial routine takes over)
constexpr uint32_t MC_SMALL = 192;  // up to this many regions CTA 0 simply runs the sequential loop
constexpr uint32_t MC_OVERFLOW = 0xFFFFFFFEu;
// global scratch (uint32): [0] k  [1] members  [2] end  [3] serial flag  [4] done ; then region / position / target per member
constexpr int MC_CTL = 8, MC_REGION = MC_CTL, MC_POS = MC_REGION + MC_BMAX, MC_TARGET = MC_POS + MC_BMAX, MC_WORDS = MC_TARGET + MC_BMAX;

__device__ __forceinline__ bool boxes_separated(const int* p, const int* q) {   // a voxel of gap along some axis
  return p[0] >= q[1] + 1 || q[0] >= p[1] + 1 || p[2] >= q[3] + 1 || q[2] >= p[3] + 1 || p[4] >= q[5] + 1 || q[4] >= p[5] + 1;
}

// apply the previous batch (if any), then build the next one; CTA 0 only
__device__ void mc_apply_and_build(const MergeArgs& a, const uint32_t* pos_of, uint32_t* mc, uint32_t R) {
  __shared__ uint8_t s_cls[MC_WINDOW];
  __shared__ uint32_t s_list[MC_BMAX];
  __shared__ int s_box[MC_BMAX][6];
  __shared__ uint32_t s_r[MC_BMAX], s_pos[MC_BMAX], s_t[MC_BMAX], s_ar[MC_BMAX], s_at[MC_BMAX], s_pt[MC_BMAX], s_slot[MC_BMAX];
  __shared__ uint8_t s_tv[MC_BMAX], s_applied[MC_BMAX];
  __shared__ uint32_t s_rec[256];
  __shared__ uint32_t s_k, s_a, s_b, s_n, s_warp[MC_THREADS / 32];
  const int tid = threadIdx.x;
  const uint32_t skip = (uint32_t)a.skip_below;

  // ---------------- apply
  const uint32_t n = mc[1], end = mc[2];
  if (tid == 0) s_k = mc[0];
  if (n > 0) {
    if (tid < (int)n) {
      const uint32_t r = mc[MC_REGION + tid], t = mc[MC_TARGET + tid];
      s_r[tid] = r; s_pos[tid] = mc[MC_POS + tid]; s_t[tid] = t; s_ar[tid] = a.area[r]; s_applied[tid] = 0;
      if (t != MC_OVERFLOW && t != r) { s_tv[tid] = a.value[t]; s_at[tid] = a.area[t]; s_pt[tid] = pos_of[t]; }
    }
    for (int i = tid; i < 256; i += blockDim.x) s_rec[i] = a.record[i];
    __syncthreads();
    if (tid < (int)n) {   // the first member with the same target carries that target's running area
      uint32_t s = tid;
      for (int m = 0; m < tid; ++m) if (s_t[m] == s_t[tid]) { s = m; break; }
      s_slot[tid] = s;
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t trunc = NONE, serial = 0;
      for (uint32_t m = 0; m < n; ++m) {
        if (trunc != NONE && s_pos[m] > trunc) break;
        const uint32_t t = s_t[m];
        if (t == MC_OVERFLOW) { trunc = s_pos[m]; serial = 1; break; }   // too many neighbours for the table: sequential routine
        s_applied[m] = 1;
        if (t == s_r[m]) continue;                       // no eligible neighbour: moved = 0, nothing changes (utils.py:330-339)
        const uint32_t s = s_slot[m], before = s_at[s], moved = s_ar[m];
        if (before == s_rec[s_tv[m]]) s_rec[s_tv[m]] += moved;   // utils.py:336-337
        s_at[s] = before + moved;                                   // utils.py:339
        // a skipped region inside the span grew over the threshold: it is a candidate when its turn comes
        if (before < skip && before + moved >= skip && s_pt[m] > s_pos[m] && s_pt[m] < end && s_pt[m] < trunc) trunc = s_pt[m];
      }
      s_k = (trunc != NONE) ? trunc : end;
      mc[3] = serial;
    }
    __syncthreads();
    if (tid < (int)n && s_applied[tid] && s_t[tid] != s_r[tid]) {
      const uint32_t r = s_r[tid], t = s_t[tid];
      a.cur[r] = t;                                      // regionmask[regionmask == r] = t
      int* bt = a.bbox + 6 * (size_t)t;
      const int* br = a.bbox + 6 * (size_t)r;
      atomicMin(&bt[0], br[0]); atomicMax(&bt[1], br[1]);
      atomicMin(&bt[2], br[2]); atomicMax(&bt[3], br[3]);
      atomicMin(&bt[4], br[4]); atomicMax(&bt[5], br[5]);
      if (s_slot[tid] == (uint32_t)tid) a.area[t] = s_at[tid];
    }
    for (int i = tid; i < 256; i += blockDim.x) a.record[i] = s_rec[i];
    __threadfence();
    __syncthreads();
  }

  // ---------------- a member the table could not hold: the sequential routine processes exactly that position
  if (mc[3]) {
    const uint32_t k = s_k;
    __syncthreads();
    merge_serial_range(a, k, k + 1);
    if (tid == 0) { s_k = k + 1; mc[3] = 0; }
    __syncthreads();
  }

  // ---------------- build
  while (true) {
    const uint32_t k = s_k;
    __syncthreads();
    if (k >= R) { if (tid == 0) { mc[0] = R; mc[1] = 0; mc[4] = 1; } return; }
    const uint32_t W = R - k < (uint32_t)MC_WINDOW ? R - k : (uint32_t)MC_WINDOW;
    if (tid == 0) { s_a = NONE; s_b = NONE; s_n = 0; }
    __syncthreads();
    for (uint32_t p = tid; p < W; p += blockDim.x) {
      const uint32_t rr = a.order[k + p];
      const uint32_t ar = a.area[rr];
      const uint8_t v = a.value[rr];
      const bool cand = (ar < a.record[v] || a.spare_value[v]) && ar >= skip;
      s_cls[p] = cand ? 1 : (ar >= skip ? 2 : 0);   // 2: a non-candidate that a record growth could turn into one
      if (cand) atomicMin(&s_a, p);
    }
    __syncthreads();
    const uint32_t first = s_a;
    if (first == NONE) {   // nobody in the window is a candidate at its turn (nothing changes while we skip them)
      if (tid == 0) s_k = k + W;
      __syncthreads();
      continue;
    }
    for (uint32_t p = tid; p < W; p += blockDim.x) if (p > first && s_cls[p] == 2) atomicMin(&s_b, p);
    __syncthreads();
    const uint32_t stop = s_b < W ? s_b : W;
    // the candidates of [first, stop) in order: every thread owns a contiguous strip of the window
    const uint32_t per = (uint32_t)MC_WINDOW / blockDim.x;
    uint32_t cnt = 0;
    for (uint32_t q = 0; q < per; ++q) { const uint32_t p = tid * per + q; cnt += (p >= first && p < stop && s_cls[p] == 1) ? 1u : 0u; }
    uint32_t inc = cnt;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if ((tid & 31) >= o) inc += v; }
    if ((tid & 31) == 31) s_warp[tid >> 5] = inc;
    __syncthreads();
    if (tid < 32) {
      uint32_t w = tid < (int)(blockDim.x >> 5) ? s_warp[tid] : 0;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, w, o); if (tid >= o) w += v; }
      if (tid < (int)(blockDim.x >> 5)) s_warp[tid] = w;
    }
    __syncthreads();
    uint32_t off = inc - cnt + ((tid >> 5) ? s_warp[(tid >> 5) - 1] : 0);
    const uint32_t total = s_warp[(blockDim.x >> 5) - 1];
    for (uint32_t q = 0; q < per; ++q) {
      const uint32_t p = tid * per + q;
      if (p >= first && p < stop && s_cls[p] == 1) { if (off <= (uint32_t)MC_BMAX) { if (off < (uint32_t)MC_BMAX) s_list[off] = p; else s_n = p; } ++off; }
    }
    __syncthreads();
    uint32_t nl = total < (uint32_t)MC_BMAX ? total : (uint32_t)MC_BMAX;
    uint32_t endp = total > (uint32_t)MC_BMAX ? s_n : stop;   // the batch ends before the first candidate that did not fit
    if (tid < (int)nl) {
      const int* bb = a.bbox + 6 * (size_t)a.order[k + s_list[tid]];
      for (int c = 0; c < 6; ++c) s_box[tid][c] = bb[c];
    }
    if (tid == 0) s_a = NONE;
    __syncthreads();
    if (tid < (int)nl) {
      bool hit = false;
      for (int i = 0; i < tid && !hit; ++i) hit = !boxes_separated(s_box[i], s_box[tid]);
      if (hit) atomicMin(&s_a, (uint32_t)tid);
    }
    __syncthreads();
    if (s_a != NONE) { nl = s_a; endp = s_list[s_a]; }   // cut before the first member that touches an earlier one (nl >= 1)
    if (tid < (int)nl) { mc[MC_REGION + tid] = a.order[k + s_list[tid]]; mc[MC_POS + tid] = k + s_list[tid]; }
    if (tid == 0) { mc[0] = k; mc[1] = nl; mc[2] = k + endp; mc[4] = 0; }
    __threadfence();
    __syncthreads();
    return;
  }
}

// one batch member: the target the sequential loop would pick for region r given the current tables
__device__ void mc_decide(const MergeArgs& a, uint32_t* mc, uint32_t m) {
  __shared__ uint32_t h_key[MC_HASH], h_cnt[MC_HASH];
  __shared__ uint32_t s_over;
  __shared__ unsigned long long s_best;
  const int tid = threadIdx.x;
  const Dim d = a.d;
  const size_t HW = (size_t)d.H * d.W;
  const uint32_t r = mc[MC_REGION + m];
  for (int i = tid; i < MC_HASH; i += blockDim.x) { h_key[i] = 0; h_cnt[i] = 0; }
  if (tid == 0) { s_over = 0; s_best = 0ull; }
  __syncthreads();
  Box b;
  {
    const int* bb = a.bbox + 6 * (size_t)r;
    b.z0 = max(bb[0] - 1, 0); b.z1 = min(bb[1] + 1, d.S);
    b.y0 = max(bb[2] - 1, 0); b.y1 = min(bb[3] + 1, d.H);
    b.x0 = max(bb[4] - 1, 0); b.x1 = min(bb[5] + 1, d.W);
  }
  const size_t n = box_volume(b);
  for (size_t t = tid; t < n; t += blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    const uint32_t o = a.rid[i];
    if (o == 0 || o > a.cap) continue;
    const uint32_t id = cur_find(a.cur, o);
    if (id == r) continue;
    bool ring = false;
    if (x > 0)       { const uint32_t q = a.rid[i - 1];   ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (x < d.W - 1) { const uint32_t q = a.rid[i + 1];   ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (y > 0)       { const uint32_t q = a.rid[i - d.W]; ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (y < d.H - 1) { const uint32_t q = a.rid[i + d.W]; ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (z > 0)       { const uint32_t q = a.rid[i - HW];  ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (z < d.S - 1) { const uint32_t q = a.rid[i + HW];  ring |= (q && q <= a.cap && cur_find(a.cur, q) == r); }
    if (!ring) continue;
    uint32_t h = (id * 2654435761u) & (MC_HASH - 1);
    int probes = 0;
    while (true) {
      const uint32_t old = atomicCAS(&h_key[h], 0u, id);
      if (old == 0u || old == id) { atomicAdd(&h_cnt[h], 1u); break; }
      h = (h + 1) & (MC_HASH - 1);
      if (++probes >= MC_HASH) { s_over = 1; break; }
    }
  }
  __syncthreads();
  for (int i = tid; i < MC_HASH; i += blockDim.x) {
    const uint32_t id = h_key[i];
    if (id == 0 || a.spare_id[id]) continue;
    atomicMax(&s_best, ((unsigned long long)h_cnt[i] << 32) | (unsigned long long)(0xFFFFFFFFu - id));
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t target = r;
    if (s_over) target = MC_OVERFLOW;
    else if (s_best != 0ull) target = 0xFFFFFFFFu - (uint32_t)(s_best & 0xFFFFFFFFull);
    mc[MC_TARGET + m] = target;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(MC_THREADS, 1) merge_loop_mc_kernel(MergeArgs a, uint32_t* pos_of, uint32_t* mc) {
  cg::grid_group grid = cg::this_grid();
  const uint32_t R = *a.d_R < a.cap ? *a.d_R : a.cap;
  if (R <= MC_SMALL || gridDim.x == 1) {   // (uniform over the grid: nobody reaches a grid-wide synchronisation)
    if (blockIdx.x == 0) merge_serial_range(a, 0, R);
    return;
  }
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < R; i += gridDim.x * blockDim.x) pos_of[a.order[i]] = i;
  if (blockIdx.x == 0 && threadIdx.x < MC_CTL) mc[threadIdx.x] = 0;
  __threadfence();
  grid.sync();
  while (true) {
    if (blockIdx.x == 0) mc_apply_and_build(a, pos_of, mc, R);
    __threadfence();
    grid.sync();
    if (mc[4]) break;
    const uint32_t n = mc[1];
    for (uint32_t m = blockIdx.x; m < n; m += gridDim.x) mc_decide(a, mc, m);
    __threadfence();
    grid.sync();
  }
}

// ---- Q5 -----------------------------------------------------------------------------------------------------
__global__ void map_labels_kernel(const uint32_t* __restrict__ rid, uint32_t* __restrict__ cur,
                                  const uint8_t* __restrict__ to_label, const uint8_t* __restrict__ spare_value,
                                  uint8_t* __restrict__ mapped, size_t n, uint32_t* __restrict__ present, uint32_t cap) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o = rid[i];
    uint8_t v = 0;
    if (o && o <= cap) {
      v = to_label[cur_find(cur, o)];
      if (spare_value[v]) v = 0;
    }
    mapped[i] = v;
    if (!present[v]) present[v] = 1;
  }
}

__global__ void debug_ids_kernel(const uint32_t* __restrict__ rid, uint32_t* __restrict__ cur, uint8_t* __restrict__ out,
                                 size_t n, int merged, uint32_t cap) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t o = rid[i];
    if (o && o <= cap && merged) o = cur_find(cur, o);
    out[i] = (uint8_t)(o & 255u);
  }
}

// ---- Q6 -----------------------------------------------------------------------------------------------------
__global__ void root_area_kernel(const uint32_t* __restrict__ parent, uint32_t* __restrict__ area, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t p = parent[i];
    if (p == NONE) continue;
    const unsigned peers = __match_any_sync(__activemask(), p);
    if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&area[p], (uint32_t)__popc(peers));
  }
}
// per label value: the root with the largest area; np.argsort(areas)[-1] -> among equal areas the highest id
__global__ void best_root_kernel(const uint8_t* __restrict__ vals, const uint32_t* __restrict__ parent,
                                 const uint32_t* __restrict__ area, unsigned long long* __restrict__ best, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (parent[i] != (uint32_t)i) continue;
    atomicMax(&best[vals[i]], ((unsigned long long)area[i] << 32) | (unsigned long long)(uint32_t)i);
  }
}
// np.unique(outmask_mapped)[1:] (utils.py:355): the smallest label value present is skipped, whatever it is
__global__ void first_present_kernel(uint32_t* __restrict__ small) {
  if (threadIdx.x == 0) {
    uint32_t f = 256;
    for (int v = 255; v >= 0; --v) if (small[W_PRESENT + v]) f = (uint32_t)v;
    small[W_FIRST] = f;
  }
}
// opens the finalisation of label `v`: gate = present and not the first value; resets the extent
__global__ void label_begin_kernel(uint32_t* small, int v) {
  if (threadIdx.x == 0) {
    small[W_GATE] = (small[W_PRESENT + v] && small[W_FIRST] != (uint32_t)v) ? 1u : 0u;
    int* bb = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(small) + B_BBOX1);
    bb[0] = bb[2] = bb[4] = 1 << 30;
    bb[1] = bb[3] = bb[5] = -1;
  }
}
// keep mask of one label's largest component -> tmp = 1 where NOT kept (the "background" to analyse), and its extent
__global__ void keep_complement_kernel(const uint8_t* __restrict__ mapped, const uint32_t* __restrict__ parent,
                                       uint8_t label, const unsigned long long* __restrict__ best,
                                       uint8_t* __restrict__ tmp, Dim d, int* __restrict__ bbox,
                                       const uint32_t* __restrict__ gate) {
  if (*gate == 0u) return;
  const uint32_t root = (uint32_t)(best[label] & 0xFFFFFFFFull);
  const size_t n = (size_t)d.S * d.H * d.W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const bool keep = mapped[i] == label && parent[i] == root;
    tmp[i] = keep ? 0 : 1;
    if (keep) {
      int x, y, z;
    voxel_zyx(d, (uint32_t)i, z, y, x);
      if (z < bbox[0]) atomicMin(&bbox[0], z);
      if (z + 1 > bbox[1]) atomicMax(&bbox[1], z + 1);
      if (y < bbox[2]) atomicMin(&bbox[2], y);
      if (y + 1 > bbox[3]) atomicMax(&bbox[3], y + 1);
      if (x < bbox[4]) atomicMin(&bbox[4], x);
      if (x + 1 > bbox[5]) atomicMax(&bbox[5], x + 1);
    }
  }
}
// complement voxels on the faces of the analysis box are connected to the outside: flag their roots
__global__ void seed_outside_kernel(const uint32_t* __restrict__ parent2, uint8_t* __restrict__ outside, Dim d, BoxSrc bs) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    if (parent2[i] == NONE) continue;
    if (z == b.z0 || z == b.z1 - 1 || y == b.y0 || y == b.y1 - 1 || x == b.x0 || x == b.x1 - 1) outside[parent2[i]] = 1;
  }
}
__global__ void paint_filled_kernel(const uint32_t* __restrict__ parent2, const uint8_t* __restrict__ outside,
                                    uint8_t label, uint8_t* __restrict__ out, Dim d, BoxSrc bs) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    const uint32_t p = parent2[i];
    if (p == NONE || !outside[p]) out[i] = label;  // kept voxel, or enclosed background
  }
}
// single-slice volumes: area_closing(area_threshold=64): 4-connected background components < 64 px are filled
__global__ void paint_area_closing_kernel(const uint32_t* __restrict__ parent2, const uint32_t* __restrict__ area,
                                          uint8_t label, uint8_t* __restrict__ out, size_t n, uint32_t threshold,
                                          const uint32_t* __restrict__ gate) {
  if (*gate == 0u) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t p = parent2[i];
    if (p == NONE || area[p] < threshold) out[i] = label;
  }
}
__global__ void gated_zero_kernel(uint32_t* __restrict__ a, size_t n, const uint32_t* __restrict__ gate) {
  if (*gate == 0u) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) a[i] = 0;
}
__global__ void gated_root_area_kernel(const uint32_t* __restrict__ parent, uint32_t* __restrict__ area, size_t n,
                                       const uint32_t* __restrict__ gate) {
  if (*gate == 0u) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t p = parent[i];
    if (p == NONE) continue;
    const unsigned peers = __match_any_sync(__activemask(), p);
    if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&area[p], (uint32_t)__popc(peers));
  }
}
__global__ void clear_outside_kernel(uint8_t* __restrict__ outside, Dim d, BoxSrc bs) {
  Box b;
  if (!resolve_box(bs, d, b)) return;
  const size_t n = box_volume(b);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    int z, y, x;
    const uint32_t i = box_voxel(b, d, t, z, y, x);
    outside[i] = 0;
  }
}

// ---- reshape (utils.py:114-129) and fusion glue (mask.py:228-230) ------------------------------------------
__device__ __forceinline__ int nn_index_f64(int n_in, int n_out, int o) {
  if (n_out <= 1) return 0;
  const double step = __ddiv_rn((double)(n_in - 1), (double)(n_out - 1));
  const double c = __dmul_rn((double)o, step);
  if (c > (double)(n_in - 1)) return -1;  // scipy mode='constant': outside -> cval 0
  int i = (int)floor(__dadd_rn(c, 0.5));
  return i < 0 ? 0 : (i > n_in - 1 ? n_in - 1 : i);
}
template <typename IT>   // uint32_t for volumes below 2^32 voxels (two 32-bit divisions per voxel), size_t otherwise
__global__ void reshape_kernel(const uint8_t* __restrict__ masks, const int32_t* __restrict__ boxes, int S, int H,
                               int W, int MH, int MW, uint8_t* __restrict__ out) {
  const size_t n = (size_t)S * H * W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const IT ii = (IT)i, row = ii / (IT)W, sl = row / (IT)H;
    const int x = (int)(ii - row * (IT)W), y = (int)(row - sl * (IT)H), s = (int)sl;
    const int32_t* b = boxes + 4 * s;
    uint8_t v = 0;
    if (y >= b[0] && y < b[2] && x >= b[1] && x < b[3]) {
      const int iy = nn_index_f64(MH, b[2] - b[0], y - b[0]);
      const int ix = nn_index_f64(MW, b[3] - b[1], x - b[1]);
      if (iy >= 0 && ix >= 0) v = masks[((size_t)s * MH + iy) * MW + ix];
    }
    out[i] = v;
  }
}
__global__ void max_u8_kernel(const uint8_t* __restrict__ a, size_t n, uint32_t* __restrict__ mx) {
  uint32_t m = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = max(m, (uint32_t)a[i]);
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(mx, m);
}
// spare = res_l.max() + 1 in uint8 arithmetic (mask.py:228), left in device memory for the post-processing
__global__ void spare_from_max_kernel(const uint32_t* __restrict__ mx, int32_t* __restrict__ spare) {
  if (threadIdx.x == 0) spare[0] = (int32_t)((mx[0] + 1u) & 0xFFu);
}
__global__ void fuse_kernel(uint8_t* __restrict__ res_l, const uint8_t* __restrict__ res_r, size_t n,
                            const int32_t* __restrict__ spare_p) {
  const uint8_t spare = (uint8_t)spare_p[0];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint8_t l = res_l[i];
    const uint8_t r = res_r[i];
    if (l == 0 && r > 0) l = spare;  // mask.py:229
    if (r == 0) l = 0;               // mask.py:230
    res_l[i] = l;
  }
}

inline int grid_for(size_t n, int block, int num_sms) {
  size_t g = (n + block - 1) / block;
  const size_t cap = (size_t)num_sms * 8;
  return (int)(g < 1 ? 1 : (g < cap ? g : cap));
}

#define LM_CUDA(x)                         \
  do {                                     \
    cudaError_t e_ = (x);                  \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

inline BoxSrc fixed_box(const Box& b) { BoxSrc s; s.fixed = b; s.dyn = nullptr; s.gate = nullptr; return s; }

// n_hint: voxels the box can hold at most (grid sizing; the kernels loop over the box they resolve on the device)
template <int CONN>
int run_ccl(const uint8_t* vals, uint32_t* parent, Dim d, const BoxSrc& bs, size_t n_hint, int num_sms, cudaStream_t st,
            int64_t* launches, int rule = 1) {
  const int g = grid_for(n_hint, 256, num_sms);   // init and merge MUST share the launch shape (32-voxel segments)
  ccl_init_kernel<<<g, 256, 0, st>>>(vals, parent, d, bs);
  ccl_merge_kernel<CONN><<<g, 256, 0, st>>>(vals, parent, d, bs, rule);
  ccl_flatten_kernel<<<g, 256, 0, st>>>(parent, d, bs);
  *launches += 3;
  return (int)cudaGetLastError();
}

uint32_t pow2_at_least(uint64_t x) {
  uint64_t p = 2;
  while (p < x) p <<= 1;
  return (uint32_t)p;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------
int PostScratch::reserve(size_t nvox) {
  if (nvox <= cap_vox) return 0;
  release();
  const size_t nb = (nvox + SCAN_BLOCK * SCAN_ITEMS - 1) / (SCAN_BLOCK * SCAN_ITEMS);
  int rc = 0;
  auto A = [&](void* pp, size_t bytes) { if (!rc) { cudaError_t e = cudaMalloc((void**)pp, bytes); if (e != cudaSuccess) rc = (int)e; } };
  A(&parent, nvox * 4); A(&parent2, nvox * 4); A(&rid, nvox * 4); A(&area2, nvox * 4);
  A(&mapped, nvox); A(&tmp, nvox); A(&outside, nvox);
  A(&block_counts, (nb + 1) * 4); A(&small, 4096 * 8);
  if (!rc) { cudaError_t e = cudaMallocHost((void**)&h_small, 4096 * 8); if (e != cudaSuccess) rc = (int)e; }
  if (!rc) { cudaError_t e = cudaMemset(outside, 0, nvox); if (e != cudaSuccess) rc = (int)e; }  // kept all-zero between uses
  if (rc) { release(); return rc; }  // capacities stay 0: the next call allocates again instead of using dangling pointers
  cap_vox = nvox;
  // region tables: sized for a speckled label map (1 region per 32 voxels); a map with more regions overflows once, the
  // device reports the count and the caller retries with tables of that size
  const uint64_t want = nvox / 32 > 65536 ? nvox / 32 : 65536;
  return reserve_regions((uint32_t)(want < nvox ? want : nvox));
}
void PostScratch::release_regions() {
  cudaFree(r_area); cudaFree(r_value); cudaFree(r_bbox); cudaFree(r_cur); cudaFree(r_order); cudaFree(r_count);
  cudaFree(r_touched); cudaFree(r_spare_id); cudaFree(r_to_label); cudaFree(r_hslot); cudaFree(sort_keys);
  cudaFree(hash_keys); cudaFree(hash_min); cudaFree(batch); cudaFree(r_pos);
  r_area = r_cur = r_order = r_count = r_touched = r_hslot = nullptr; r_value = r_spare_id = r_to_label = nullptr; r_bbox = nullptr;
  sort_keys = hash_keys = nullptr; hash_min = nullptr; batch = nullptr; r_pos = nullptr;
  cap_regions = 0; hash_cap = 0; sort_cap = 0;
}
int PostScratch::reserve_regions(uint32_t R) {
  if (R <= cap_regions && cap_regions) return 0;
  release_regions();
  const size_t c = (size_t)R + 1;
  const uint32_t hc = pow2_at_least(2 * (uint64_t)c), sc = pow2_at_least(c);
  int rc = 0;
  auto A = [&](void* pp, size_t bytes) { if (!rc) { cudaError_t e = cudaMalloc((void**)pp, bytes); if (e != cudaSuccess) rc = (int)e; } };
  A(&r_area, c * 4); A(&r_value, c); A(&r_bbox, c * 6 * 4); A(&r_cur, c * 4); A(&r_order, c * 4); A(&r_count, c * 4);
  A(&r_touched, c * 4); A(&r_spare_id, c); A(&r_to_label, c); A(&r_hslot, c * 4);
  A(&sort_keys, (size_t)sc * 8); A(&hash_keys, (size_t)hc * 8); A(&hash_min, (size_t)hc * 4);
  A(&r_pos, c * 4); A(&batch, (size_t)MC_WORDS * 4);
  if (rc) { release_regions(); return rc; }
  cap_regions = R; hash_cap = hc; sort_cap = sc;
  return 0;
}
void PostScratch::release() {
  cudaFree(parent); cudaFree(parent2); cudaFree(rid); cudaFree(area2); cudaFree(mapped); cudaFree(tmp); cudaFree(outside);
  cudaFree(block_counts); cudaFree(small);
  if (h_small) cudaFreeHost(h_small);
  parent = parent2 = rid = area2 = nullptr; mapped = tmp = outside = nullptr; block_counts = nullptr; small = nullptr; h_small = nullptr;
  release_regions();
  cap_vox = 0;
}

int ccl_slab_device(const uint8_t* d_labels, uint32_t* d_parent, int S, int H, int W, int z_lo, int z_hi, int rule, int num_sms,
                    cudaStream_t st, int64_t* launches) {
  if (z_hi <= z_lo) return 0;
  const Dim d{S, H, W};
  const Box slab{z_lo, z_hi, 0, H, 0, W};
  const BoxSrc bs = fixed_box(slab);
  const size_t n = (size_t)(z_hi - z_lo) * H * W;
  const int g = grid_for(n, 256, num_sms);
  ccl_init_kernel<<<g, 256, 0, st>>>(d_labels, d_parent, d, bs);
  ccl_merge_kernel<26><<<g, 256, 0, st>>>(d_labels, d_parent, d, bs, rule);
  *launches += 2;
  return (int)cudaGetLastError();
}

int ccl_join_slabs_device(const uint8_t* d_labels, uint32_t* d_parent, int S, int H, int W, const int* first_slices, int n_bounds,
                          int num_sms, cudaStream_t st, int64_t* launches) {
  const Dim d{S, H, W};
  const Box full{0, S, 0, H, 0, W};
  if (n_bounds > 16) return -24;
  if (n_bounds > 0) {
    SlabBounds sb{};
    sb.n = n_bounds;
    for (int i = 0; i < n_bounds; ++i) sb.z[i] = first_slices[i];
    ccl_join_slabs_kernel<<<grid_for((size_t)n_bounds * H * W, 256, num_sms), 256, 0, st>>>(d_labels, d_parent, d, sb);
    *launches += 1;
  }
  ccl_flatten_kernel<<<grid_for((size_t)S * H * W, 256, num_sms), 256, 0, st>>>(d_parent, d, fixed_box(full));
  *launches += 1;
  return (int)cudaGetLastError();
}

int postprocess_device(PostScratch& ws, const uint8_t* d_labels, int S, int H, int W, const int32_t* spare, int n_spare,
                       const int32_t* d_spare, int n_d_spare, int skip_below, int max_label, uint8_t* d_out, int num_sms,
                       cudaStream_t st, int64_t* launches, uint32_t* parent_in) {
  const size_t n = (size_t)S * H * W;
  if (n == 0) return 0;
  if (n >= 0xFFFFFFF0ull) return -20;
  if (n_spare < 0 || n_d_spare < 0 || n_spare + n_d_spare > MAX_SPARE) return -23;
  int rc = ws.reserve(n);
  if (rc) return rc;
  const Dim d{S, H, W};
  const Box full{0, S, 0, H, 0, W};
  const BoxSrc fullsrc = fixed_box(full);
  const int g = grid_for(n, 256, num_sms);
  uint32_t* d_small = reinterpret_cast<uint32_t*>(ws.small);
  uint8_t* small_b = reinterpret_cast<uint8_t*>(ws.small);
  uint32_t* d_record = d_small + W_RECORD;
  uint32_t* d_present = d_small + W_PRESENT;
  const uint32_t* d_gate = d_small + W_GATE;
  uint8_t* d_spare_value = small_b + B_SPARE_VALUE;
  unsigned long long* d_best = reinterpret_cast<unsigned long long*>(small_b + B_BEST);
  int* d_bbox1 = reinterpret_cast<int*>(small_b + B_BBOX1);
  const uint32_t cap = ws.cap_regions;
  ws.want_regions = 0;

  SpareArgs sp{};
  sp.n = n_spare;
  for (int i = 0; i < n_spare; ++i) sp.v[i] = spare[i];
  sp.d_extra = d_spare; sp.n_extra = n_d_spare;
  post_setup_kernel<<<1, 256, 0, st>>>(d_small, sp, ws.clear_sticky ? 1 : 0);
  ws.clear_sticky = false;

  // Q1: components + canonical ids (R stays on the device: d_small[W_R]); parent_in: the flattened union-find of a
  // slab-wise labelling that the caller has already joined (ccl_slab_device / ccl_join_slabs_device)
  uint32_t* const parent1 = parent_in ? parent_in : ws.parent;
  if (!parent_in) {
    rc = run_ccl<26>(d_labels, ws.parent, d, fullsrc, n, num_sms, st, launches, ws.ccl_rule);
    if (rc) return rc;
  }
  const int nb = (int)((n + SCAN_BLOCK * SCAN_ITEMS - 1) / (SCAN_BLOCK * SCAN_ITEMS));
  roots_count_kernel<<<nb, SCAN_BLOCK, 0, st>>>(parent1, n, ws.block_counts);
  scan_blocks_kernel<<<1, 1024, 0, st>>>(ws.block_counts, nb, d_small + W_R);
  roots_assign_kernel<<<nb, SCAN_BLOCK, 0, st>>>(parent1, n, ws.block_counts, ws.rid);

  // Q2: region tables
  const int gr = grid_for((size_t)cap + 1, 256, num_sms);
  region_init_kernel<<<gr, 256, 0, st>>>(d_small, cap, ws.r_area, ws.r_count, ws.r_value, ws.r_bbox, ws.r_cur, ws.r_to_label,
                                         ws.r_spare_id);
  region_stats_kernel<<<g, 256, 0, st>>>(d_labels, parent1, ws.rid, d, cap, ws.r_area, ws.r_value, ws.r_bbox);
  // Q3: ascending (area, id) order, per-label records, region -> label table
  region_sort_kernel<<<1, 1024, 0, st>>>(d_small, cap, ws.r_area, reinterpret_cast<unsigned long long*>(ws.sort_keys), ws.r_order);
  LM_CUDA(cudaMemsetAsync(ws.hash_keys, 0xFF, (size_t)ws.hash_cap * 8, st));
  LM_CUDA(cudaMemsetAsync(ws.hash_min, 0xFF, (size_t)ws.hash_cap * 4, st));
  record_insert_kernel<<<gr, 256, 0, st>>>(d_small, cap, ws.r_area, ws.r_value, reinterpret_cast<unsigned long long*>(ws.hash_keys),
                                           ws.hash_min, ws.hash_cap - 1, ws.r_hslot);
  record_lookup_kernel<<<gr, 256, 0, st>>>(d_small, cap, ws.r_value, ws.hash_min, ws.r_hslot, ws.r_to_label);
  // Q4
  MergeArgs ma;
  ma.rid = ws.rid; ma.cur = ws.r_cur; ma.area = ws.r_area; ma.value = ws.r_value; ma.bbox = ws.r_bbox;
  ma.record = d_record; ma.order = ws.r_order; ma.count = ws.r_count; ma.touched = ws.r_touched;
  ma.spare_value = d_spare_value; ma.spare_id = ws.r_spare_id; ma.d_R = d_small + W_R; ma.cap = cap;
  ma.skip_below = skip_below; ma.d = d;
  // many CTAs when the device can co-schedule a grid (cooperative launch), else the one-CTA loop
  bool launched = false;
  if (ws.merge_ctas != 1) {
    static std::atomic<int> coop_ok{-1};   // -1 unknown, 0 no, 1 yes (per process: every engine device is an H100)
    if (coop_ok.load() < 0) {
      int dev = 0, v = 0;
      if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrCooperativeLaunch, dev) == cudaSuccess) coop_ok.store(v ? 1 : 0);
      else coop_ok.store(0);
    }
    if (coop_ok.load() == 1) {
      uint32_t* pos_of = ws.r_pos;
      uint32_t* mc = ws.batch;
      void* args[] = {(void*)&ma, (void*)&pos_of, (void*)&mc};
      const int ctas = ws.merge_ctas > 1 ? (ws.merge_ctas < num_sms ? ws.merge_ctas : num_sms) : num_sms;
      const cudaError_t ce = cudaLaunchCooperativeKernel((void*)merge_loop_mc_kernel, dim3(ctas), dim3(MC_THREADS), args, 0, st);
      if (ce == cudaSuccess) launched = true;
      else { cudaGetLastError(); coop_ok.store(0); }
    }
  }
  if (!launched) merge_loop_kernel<<<1, 1024, 0, st>>>(ma);
  // Q5
  map_labels_kernel<<<g, 256, 0, st>>>(ws.rid, ws.r_cur, ws.r_to_label, d_spare_value, ws.mapped, n, d_present, cap);
  *launches += 11;

  // R and the overflow flag travel to the pinned mirror now; the host looks at them in postprocess_finish
  LM_CUDA(cudaMemcpyAsync(ws.h_small, d_small, 8, cudaMemcpyDeviceToHost, st));

  if (ws.debug_stage == 1) { LM_CUDA(cudaMemcpyAsync(d_out, ws.mapped, n, cudaMemcpyDeviceToDevice, st)); return 0; }
  if (ws.debug_stage == 2 || ws.debug_stage == 3) {
    debug_ids_kernel<<<g, 256, 0, st>>>(ws.rid, ws.r_cur, d_out, n, ws.debug_stage == 3, cap);
    return (int)cudaGetLastError();
  }
  // Q6
  LM_CUDA(cudaMemsetAsync(d_out, 0, n, st));
  LM_CUDA(cudaMemsetAsync(ws.outside, 0, n, st));
  rc = run_ccl<26>(ws.mapped, ws.parent, d, fullsrc, n, num_sms, st, launches, ws.ccl_rule);
  if (rc) return rc;
  LM_CUDA(cudaMemsetAsync(ws.area2, 0, n * 4, st));
  root_area_kernel<<<g, 256, 0, st>>>(ws.parent, ws.area2, n);
  best_root_kernel<<<g, 256, 0, st>>>(ws.mapped, ws.parent, ws.area2, d_best, n);
  first_present_kernel<<<1, 32, 0, st>>>(d_small);
  *launches += 3;

  // the labels to finalise: 1..max_label when the caller knows a bound (no host round trip; absent labels cost a few
  // empty launches), otherwise the values that occur (ONE synchronisation)
  bool todo[256];
  memset(todo, 0, sizeof(todo));
  if (max_label >= 0) {
    for (int v = 1; v <= max_label && v < 256; ++v) todo[v] = true;  // 0, when present, is always np.unique(...)[0]
  } else {
    uint32_t* h_present = reinterpret_cast<uint32_t*>(ws.h_small) + 16;
    LM_CUDA(cudaMemcpyAsync(h_present, d_present, 256 * 4, cudaMemcpyDeviceToHost, st));
    LM_CUDA(cudaStreamSynchronize(st));
    for (int v = 0; v < 256; ++v) todo[v] = h_present[v] != 0;
  }
  BoxSrc boxsrc;
  boxsrc.fixed = full; boxsrc.dyn = d_bbox1; boxsrc.gate = d_gate;
  BoxSrc gated_full = fullsrc;
  gated_full.gate = d_gate;
  for (int v = 0; v < 256; ++v) {
    if (!todo[v]) continue;
    label_begin_kernel<<<1, 32, 0, st>>>(d_small, v);   // gate: present and not np.unique(...)[0] (utils.py:355)
    keep_complement_kernel<<<g, 256, 0, st>>>(ws.mapped, ws.parent, (uint8_t)v, d_best, ws.tmp, d, d_bbox1, d_gate);
    *launches += 2;
    if (S == 1) {
      rc = run_ccl<4>(ws.tmp, ws.parent2, d, gated_full, n, num_sms, st, launches);
      if (rc) return rc;
      gated_zero_kernel<<<g, 256, 0, st>>>(ws.area2, n, d_gate);
      gated_root_area_kernel<<<g, 256, 0, st>>>(ws.parent2, ws.area2, n, d_gate);
      paint_area_closing_kernel<<<g, 256, 0, st>>>(ws.parent2, ws.area2, (uint8_t)v, d_out, n, 64u, d_gate);
      *launches += 3;
    } else {
      rc = run_ccl<6>(ws.tmp, ws.parent2, d, boxsrc, n, num_sms, st, launches);
      if (rc) return rc;
      seed_outside_kernel<<<g, 256, 0, st>>>(ws.parent2, ws.outside, d, boxsrc);
      paint_filled_kernel<<<g, 256, 0, st>>>(ws.parent2, ws.outside, (uint8_t)v, d_out, d, boxsrc);
      clear_outside_kernel<<<g, 256, 0, st>>>(ws.outside, d, boxsrc);
      *launches += 3;
    }
  }
  return (int)cudaGetLastError();
}

int postprocess_finish(PostScratch& ws) {
  if (!ws.h_small) return 0;
  uint32_t* h = reinterpret_cast<uint32_t*>(ws.h_small);
  ws.clear_sticky = true;   // the next run starts a new observation window
  ws.last_regions = h[W_MAXR];
  if (h[W_OVERFLOW]) {
    ws.want_regions = h[W_MAXR] + h[W_MAXR] / 8 + 1024;
    h[W_OVERFLOW] = 0;
    return 1;
  }
  return 0;
}

__global__ void select_root_kernel(const uint32_t* __restrict__ parent, uint32_t root, uint8_t* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = (parent[i] != NONE && parent[i] == root) ? 1 : 0;
}
__global__ void binarize_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = in[i] ? 1 : 0;
}

// utils.keep_largest_connected_component (utils.py:390-404): full-connectivity components of a binary mask, the
// largest one kept (np.argsort(areas)[-1]: among equal areas the highest id, i.e. the last in raster order).
int keep_largest_component_device(PostScratch& ws, const uint8_t* d_mask, int S, int H, int W, uint8_t* d_out, int num_sms,
                                  cudaStream_t st) {
  const size_t n = (size_t)S * H * W;
  if (n == 0) return 0;
  if (n >= 0xFFFFFFF0ull) return -20;
  int rc = ws.reserve(n);
  if (rc) return rc;
  const Dim d{S, H, W};
  const Box full{0, S, 0, H, 0, W};
  const int g = grid_for(n, 256, num_sms);
  int64_t launches = 0;
  binarize_kernel<<<g, 256, 0, st>>>(d_mask, ws.tmp, n);
  rc = run_ccl<26>(ws.tmp, ws.parent, d, fixed_box(full), n, num_sms, st, &launches, ws.ccl_rule);
  if (rc) return rc;
  LM_CUDA(cudaMemsetAsync(ws.area2, 0, n * 4, st));
  unsigned long long* d_best = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(ws.small) + B_BEST);
  LM_CUDA(cudaMemsetAsync(d_best, 0, 256 * 8, st));
  root_area_kernel<<<g, 256, 0, st>>>(ws.parent, ws.area2, n);
  best_root_kernel<<<g, 256, 0, st>>>(ws.tmp, ws.parent, ws.area2, d_best, n);
  unsigned long long* h_best = reinterpret_cast<unsigned long long*>(ws.h_small) + 1024;
  LM_CUDA(cudaMemcpyAsync(h_best, d_best + 1, 8, cudaMemcpyDeviceToHost, st));
  LM_CUDA(cudaStreamSynchronize(st));  // the reference raises on an empty mask: the host must know
  if (*h_best == 0ull) { LM_CUDA(cudaMemsetAsync(d_out, 0, n, st)); return -21; }  // empty mask: argsort of []
  select_root_kernel<<<g, 256, 0, st>>>(ws.parent, (uint32_t)(*h_best & 0xFFFFFFFFull), d_out, n);
  return (int)cudaGetLastError();
}

int reshape_device(const uint8_t* d_masks, const int32_t* d_boxes, int S, int H, int W, int MH, int MW, uint8_t* d_out,
                   int num_sms, cudaStream_t st) {
  const size_t n = (size_t)S * H * W;
  if (n < 0xFFFFFFF0ull) reshape_kernel<uint32_t><<<grid_for(n, 256, num_sms), 256, 0, st>>>(d_masks, d_boxes, S, H, W, MH, MW, d_out);
  else reshape_kernel<size_t><<<grid_for(n, 256, num_sms), 256, 0, st>>>(d_masks, d_boxes, S, H, W, MH, MW, d_out);
  return (int)cudaGetLastError();
}

int fuse_device(uint8_t* d_res_l, const uint8_t* d_res_r, size_t n, uint32_t* d_scratch, int32_t* d_spare_out, int num_sms,
                cudaStream_t st) {
  LM_CUDA(cudaMemsetAsync(d_scratch, 0, 4, st));
  max_u8_kernel<<<grid_for(n, 256, num_sms), 256, 0, st>>>(d_res_l, n, d_scratch);
  spare_from_max_kernel<<<1, 32, 0, st>>>(d_scratch, d_spare_out);
  fuse_kernel<<<grid_for(n, 256, num_sms), 256, 0, st>>>(d_res_l, d_res_r, n, d_spare_out);
  return (int)cudaGetLastError();
}

}  // namespace lm
