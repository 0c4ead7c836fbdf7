// Size distributions of the connected clusters of low-attenuation (LAA) voxels per label (lm_laa_clusters_dev, DESIGN §4.7).
//
// Passes, each grid-stride over the volume:
//   1. map        reads the mask as 16-byte vectors and the value only under a non-zero label; writes map_l = laa ? mask : 0
//                 (the per-label rows: equal-value labelling never crosses a label boundary) and map_u = laa ? 1 : 0 (the
//                 union row)
//   2. labelling  postproc.cu's union-find (ccl_volume_device) of map_l, later of map_u: parent = the component's minimum
//                 linear index
//   3. area       area[parent[i]] += 1 per LAA voxel, aggregated per warp with __match_any_sync (a large bulla would
//                 otherwise put every atomic on one address)
//   4. histogram  per root: row = its map value (or 256), size = area[root]; sizes below kClusterDense count in a dense
//                 [257][4096] array (the sizes below kSmallSizes privatised in shared memory), larger ones go to an
//                 overflow list of (row, size)
// Passes 2-4 run once for map_l and once for map_u.  The host then reads each row's dense extent, copies those bins and
// the overflow list, and compacts them into (size, count) pairs: sorted overflow entries after the scanned dense bins.
// zone_sizes (lm_zone_sizes_dev, DESIGN §4.9) runs passes 2-4 and the compaction once, 26-connected, on a caller's
// texture level map: the size-zone matrix, row = level; zone_sizes_plane (lm_zone_sizes_plane_dev, DESIGN §4.18) the same
// 8-connected within the planes normal to an axis, on the map permuted so that those planes are slices.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/lungmask_b200.h"
#include "clusters.cuh"
#include "mask_chunk.cuh"
#include "postproc.cuh"

namespace lm {
namespace {

constexpr int kThreads = 512;
constexpr int kSmallSizes = 32;        // sizes 1..31 of every row in shared memory: 257 x 32 x 4 B = 32.9 KB
constexpr uint32_t kNone = 0xFFFFFFFFu;

typedef unsigned long long u64;

// value < t in the volume's type: integers unclipped, float16 / bfloat16 widened to float32; NaN compares false
template <typename T> __device__ __forceinline__ bool below(T x, int t) {
  if constexpr (std::is_integral<T>::value) return (long long)x < (long long)t;
  else if constexpr (std::is_same<T, __half>::value) return __half2float(x) < (float)t;
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat162float(x) < (float)t;
  else return x < (T)t;
}

// ---- 1. LAA maps ------------------------------------------------------------------------------------------------------
// The maps are padded to whole 16-voxel chunks (zero past n), so every chunk is stored as one 16-byte vector.
template <typename T>
__global__ void __launch_bounds__(kThreads) laa_map_kernel(const T* __restrict__ vol, const uint8_t* __restrict__ mask, size_t n,
                                                           int t, uint8_t* __restrict__ map_l, uint8_t* __restrict__ map_u) {
  const size_t chunks = (n + kChunk - 1) / kChunk;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < chunks; c += (size_t)gridDim.x * blockDim.x) {
    const size_t base = c * kChunk;
    const uint4 lab = load_labels(mask, base, n);
    unsigned wl[4] = {0, 0, 0, 0}, wu[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < kChunk; ++k) {
      const int l = label_at(lab, k);
      if (l && below(vol[base + k], t)) {
        wl[k >> 2] |= (unsigned)l << (8 * (k & 3));
        wu[k >> 2] |= 1u << (8 * (k & 3));
      }
    }
    reinterpret_cast<uint4*>(map_l)[c] = make_uint4(wl[0], wl[1], wl[2], wl[3]);
    reinterpret_cast<uint4*>(map_u)[c] = make_uint4(wu[0], wu[1], wu[2], wu[3]);
  }
}

// ---- 3. cluster sizes ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) cluster_area_kernel(const uint32_t* __restrict__ parent, uint32_t* __restrict__ area,
                                                                size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t p = parent[i];
    if (p == kNone) continue;
    const unsigned peers = __match_any_sync(__activemask(), p);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&area[p], (uint32_t)__popc(peers));
  }
}

// ---- 4. size histogram ------------------------------------------------------------------------------------------------
// fixed_row 0: the row of a root is its map value; otherwise fixed_row.  row_max[r]: the largest dense size seen in row r
// (the host copies dense bins 0..row_max[r] only).  over: (row << 32 | size) for sizes >= kClusterDense, *n_over entries.
__global__ void __launch_bounds__(kThreads) cluster_hist_kernel(const uint32_t* __restrict__ parent, const uint32_t* __restrict__ area,
                                                                const uint8_t* __restrict__ map, size_t n, int fixed_row,
                                                                uint32_t* __restrict__ dense, uint32_t* __restrict__ row_max,
                                                                u64* __restrict__ over, uint32_t* __restrict__ n_over) {
  __shared__ uint32_t s_small[kClusterRows * kSmallSizes];
  for (int i = threadIdx.x; i < kClusterRows * kSmallSizes; i += blockDim.x) s_small[i] = 0;
  __syncthreads();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (parent[i] != (uint32_t)i) continue;
    const int row = fixed_row ? fixed_row : (int)map[i];
    const uint32_t s = area[i];
    if (s < (uint32_t)kSmallSizes) {
      // speckle: most lanes of a warp hold size-1 (or size-2) roots of one row
      const unsigned key = (unsigned)row * kSmallSizes + s;
      const unsigned peers = __match_any_sync(__activemask(), key);
      if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&s_small[key], (uint32_t)__popc(peers));
    } else if (s < (uint32_t)kClusterDense) {
      atomicAdd(&dense[(size_t)row * kClusterDense + s], 1u);
      atomicMax(&row_max[row], s);
    } else {
      over[atomicAdd(n_over, 1u)] = ((u64)row << 32) | s;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kClusterRows * kSmallSizes; i += blockDim.x) {
    if (!s_small[i]) continue;
    const int row = i / kSmallSizes, s = i % kSmallSizes;
    atomicAdd(&dense[(size_t)row * kClusterDense + s], s_small[i]);
    atomicMax(&row_max[row], (uint32_t)s);
  }
}

// ---- in-plane zones --------------------------------------------------------------------------------------------------------
// out = the (n0,n1,n2) map with `axis` (1 or 2) moved to the front: (n1,n0,n2) or (n2,n0,n1), so that the planes normal to
// `axis` become slices.  Zone sizes do not change under the permutation.
__global__ void __launch_bounds__(kThreads) plane_permute_kernel(const uint8_t* __restrict__ in, int n0, int n1, int n2, int axis,
                                                                 uint8_t* __restrict__ out) {
  const size_t n = (size_t)n0 * n1 * n2;
  const uint32_t m1 = (uint32_t)n0, m2 = (uint32_t)(axis == 1 ? n2 : n1);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    const uint32_t c = (uint32_t)(t % m2), r = (uint32_t)(t / m2), b = r % m1, a = r / m1;   // out[a][b][c]
    const size_t src = axis == 1 ? ((size_t)b * n1 + a) * n2 + c : ((size_t)b * n1 + c) * n2 + a;
    out[t] = in[src];
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------------
#define SC(x)                                   \
  do {                                          \
    const cudaError_t e_ = (x);                 \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Device work area (byte offsets into ClusterWork::d).
struct ClusterDev {
  uint32_t *parent, *area;   // [n]
  uint8_t *map_l, *map_u;    // [n rounded up to 16]
  uint32_t* dense;           // [257][kClusterDense]
  uint32_t* row_max;         // [257]
  uint32_t* n_over;          // [1]
  u64* over;                 // [over_cap]
};

// Each labelling has at most n / kClusterDense clusters of kClusterDense voxels or more, and there are at most two
// labellings.
size_t over_cap(size_t n) { return 2 * (n / kClusterDense) + 2; }

// Carves the work area; returns its size (d == nullptr: size only).  maps: with the two LAA maps (laa_clusters);
// zone_sizes labels the caller's map.
size_t layout(char* d, size_t n, bool maps, ClusterDev* g) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = d ? d + off : nullptr; off += align256(bytes); return p; };
  const size_t padded = maps ? (n + kChunk - 1) / kChunk * kChunk : 0;
  g->parent = (uint32_t*)take(n * 4);
  g->area = (uint32_t*)take(n * 4);
  g->map_l = maps ? (uint8_t*)take(padded) : nullptr;
  g->map_u = maps ? (uint8_t*)take(padded) : nullptr;
  g->dense = (uint32_t*)take((size_t)kClusterRows * kClusterDense * 4);
  g->row_max = (uint32_t*)take(kClusterRows * 4);
  g->n_over = (uint32_t*)take(4);
  g->over = (u64*)take(over_cap(n) * 8);
  return off;
}

template <typename K>
int grid_for(K kernel, size_t smem, size_t work, int num_sms) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const size_t need = (work + kThreads - 1) / kThreads;
  return (int)std::max<size_t>(std::min((size_t)per_sm * num_sms, need), 1);
}

template <typename T>
int launch_map(const void* vol, const uint8_t* mask, size_t n, int t, const ClusterDev& g, int num_sms, cudaStream_t st) {
  const size_t chunks = (n + kChunk - 1) / kChunk;
  laa_map_kernel<T><<<grid_for(laa_map_kernel<T>, 0, chunks, num_sms), kThreads, 0, st>>>(static_cast<const T*>(vol), mask, n, t,
                                                                                          g.map_l, g.map_u);
  return (int)cudaGetLastError();
}

int map_pass(int dtype, const void* vol, const uint8_t* mask, size_t n, int t, const ClusterDev& g, int num_sms, cudaStream_t st) {
  switch (dtype) {
    case LM_DTYPE_U8: return launch_map<uint8_t>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_I8: return launch_map<int8_t>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_I16: return launch_map<int16_t>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_I32: return launch_map<int32_t>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_I64: return launch_map<int64_t>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_F16: return launch_map<__half>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_BF16: return launch_map<__nv_bfloat16>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_F32: return launch_map<float>(vol, mask, n, t, g, num_sms, st);
    case LM_DTYPE_F64: return launch_map<double>(vol, mask, n, t, g, num_sms, st);
    default: return -1;
  }
}

// Clears the size histogram of the work area.
int clear_histogram(const ClusterDev& g, cudaStream_t st) {
  SC(cudaMemsetAsync(g.dense, 0, (size_t)kClusterRows * kClusterDense * 4, st));
  SC(cudaMemsetAsync(g.row_max, 0, kClusterRows * 4, st));
  SC(cudaMemsetAsync(g.n_over, 0, 4, st));
  return 0;
}

// Passes 2-4 on one map: the equal-value components, their sizes, and their count in the histogram at row = the map
// value (fixed_row 0) or fixed_row.
int count_components(const ClusterDev& g, const uint8_t* map, int n0, int n1, int n2, int conn, int fixed_row, int num_sms,
                     cudaStream_t st, int64_t* launches) {
  const size_t n = (size_t)n0 * n1 * n2;
  const int lrc = ccl_volume_device(map, g.parent, n0, n1, n2, conn, num_sms, st, launches);
  if (lrc) return lrc;
  SC(cudaMemsetAsync(g.area, 0, n * 4, st));
  cluster_area_kernel<<<grid_for(cluster_area_kernel, 0, n, num_sms), kThreads, 0, st>>>(g.parent, g.area, n);
  cluster_hist_kernel<<<grid_for(cluster_hist_kernel, 0, n, num_sms), kThreads, 0, st>>>(g.parent, g.area, map, n, fixed_row,
                                                                                        g.dense, g.row_max, g.over, g.n_over);
  SC(cudaGetLastError());
  *launches += 2;
  return 0;
}

// The histogram of rows 1..256 as (size, count) pairs: reads each row's dense extent, copies those bins and the
// overflow list, and writes sorted overflow entries after the scanned dense bins.  Synchronises `st` twice.
int compact_histogram(const ClusterDev& g, const LaaClustersOut& out, cudaStream_t st) {
  for (int r = 0; r < kClusterRows; ++r) out.laa_voxels[r] = out.n_clusters[r] = out.n_pairs[r] = 0;
  // the extent of every row's dense bins and the overflow count, then only those bins and entries
  uint32_t row_max[kClusterRows], n_over = 0;
  SC(cudaMemcpyAsync(row_max, g.row_max, sizeof(row_max), cudaMemcpyDeviceToHost, st));
  SC(cudaMemcpyAsync(&n_over, g.n_over, 4, cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  size_t first[kClusterRows + 1];   // row r's bins 0..row_max[r] are dense[first[r] .. first[r + 1])
  first[0] = 0;
  for (int r = 0; r < kClusterRows; ++r) first[r + 1] = first[r] + (row_max[r] ? (size_t)row_max[r] + 1 : 0);
  std::vector<uint32_t> dense(first[kClusterRows]);
  for (int r = 1; r < kClusterRows; ++r)
    if (row_max[r])
      SC(cudaMemcpyAsync(&dense[first[r]], g.dense + (size_t)r * kClusterDense, ((size_t)row_max[r] + 1) * 4,
                         cudaMemcpyDeviceToHost, st));
  std::vector<u64> over(n_over);
  if (n_over) SC(cudaMemcpyAsync(over.data(), g.over, (size_t)n_over * 8, cudaMemcpyDeviceToHost, st));
  SC(cudaStreamSynchronize(st));
  std::sort(over.begin(), over.end());   // by row, then size

  size_t k = 0, o = 0;
  for (int r = 1; r < kClusterRows; ++r) {
    int64_t vox = 0, clusters = 0, pairs = 0;
    auto emit = [&](int64_t size, int64_t count) {
      if (k < out.max_pairs) { out.sizes[k] = size; out.counts[k] = count; }
      ++k;
      ++pairs;
      clusters += count;
      vox += size * count;
    };
    for (uint32_t s = 1; s <= row_max[r]; ++s)
      if (dense[first[r] + s]) emit(s, dense[first[r] + s]);
    while (o < over.size() && (int)(over[o] >> 32) == r) {
      const uint32_t s = (uint32_t)over[o];
      int64_t c = 0;
      while (o < over.size() && over[o] == (((u64)r << 32) | s)) { ++c; ++o; }
      emit(s, c);
    }
    out.laa_voxels[r] = vox;
    out.n_clusters[r] = clusters;
    out.n_pairs[r] = pairs;
  }
  return k <= out.max_pairs ? 0 : -1;   // unreachable: max_pairs >= laa_max_pairs(n) bounds k
}

}  // namespace

size_t laa_max_pairs(size_t n_voxels) {
  // ceil(sqrt(n)), exact for every size_t
  unsigned __int128 s = (unsigned __int128)sqrtl((long double)n_voxels);
  while (s * s < n_voxels) ++s;
  while (s > 0 && (s - 1) * (s - 1) >= n_voxels) --s;
  return (size_t)(32 * s + 256);
}

int ClusterWork::reserve(size_t bytes) {
  if (bytes <= d_bytes) return 0;
  release();
  const cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) { d = nullptr; return (int)e; }
  d_bytes = bytes;
  return 0;
}

void ClusterWork::release() {
  if (d) cudaFree(d);
  d = nullptr;
  d_bytes = 0;
}

int laa_clusters(ClusterWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2, int threshold,
                 int conn, const LaaClustersOut& out, int num_sms, cudaStream_t st, int64_t* launches) {
  if (conn != 4 && conn != 6 && conn != 26) return -1;
  const size_t n = (size_t)n0 * n1 * n2;
  for (int r = 0; r < kClusterRows; ++r) out.laa_voxels[r] = out.n_clusters[r] = out.n_pairs[r] = 0;
  ClusterDev g;
  SC((cudaError_t)w.reserve(layout(nullptr, n, true, &g)));
  layout(static_cast<char*>(w.d), n, true, &g);

  const int crc = clear_histogram(g, st);
  if (crc) return crc;
  const int rc = map_pass(dtype, d_vol, d_mask, n, threshold, g, num_sms, st);
  if (rc) return rc;
  ++*launches;
  for (int pass = 0; pass < 2; ++pass) {
    const int lrc = count_components(g, pass ? g.map_u : g.map_l, n0, n1, n2, conn, pass ? 256 : 0, num_sms, st, launches);
    if (lrc) return lrc;
  }
  return compact_histogram(g, out, st);
}

namespace {
// zone_sizes (axis < 0: 26-connected) and zone_sizes_plane (8-connected within the planes normal to axis; axes 1 and 2
// label the permuted map in map_l).
int zones_of(ClusterWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int axis, int64_t* n_pairs, int64_t* sizes,
             int64_t* counts, size_t max_pairs, int num_sms, cudaStream_t st, int64_t* launches) {
  const size_t n = (size_t)n0 * n1 * n2;
  const bool permute = axis > 0;
  ClusterDev g;
  SC((cudaError_t)w.reserve(layout(nullptr, n, permute, &g)));
  layout(static_cast<char*>(w.d), n, permute, &g);
  const int crc = clear_histogram(g, st);
  if (crc) return crc;
  const uint8_t* map = d_levels;
  int m0 = n0, m1 = n1, m2 = n2;
  if (permute) {
    plane_permute_kernel<<<grid_for(plane_permute_kernel, 0, n, num_sms), kThreads, 0, st>>>(d_levels, n0, n1, n2, axis, g.map_l);
    SC(cudaGetLastError());
    ++*launches;
    map = g.map_l;
    m0 = axis == 1 ? n1 : n2, m1 = n0, m2 = axis == 1 ? n2 : n1;
  }
  const int lrc = count_components(g, map, m0, m1, m2, axis < 0 ? 26 : 8, 0, num_sms, st, launches);
  if (lrc) return lrc;
  int64_t voxels[kClusterRows], zones[kClusterRows], pairs[kClusterRows];
  const int rc = compact_histogram(g, {voxels, zones, pairs, sizes, counts, max_pairs}, st);
  for (int r = 0; r < 256; ++r) n_pairs[r] = pairs[r];   // row 256 (the union) stays empty: fixed_row is 0
  return rc;
}
}  // namespace

int zone_sizes(ClusterWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int64_t* n_pairs, int64_t* sizes,
               int64_t* counts, size_t max_pairs, int num_sms, cudaStream_t st, int64_t* launches) {
  return zones_of(w, d_levels, n0, n1, n2, -1, n_pairs, sizes, counts, max_pairs, num_sms, st, launches);
}

int zone_sizes_plane(ClusterWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int axis, int64_t* n_pairs, int64_t* sizes,
                     int64_t* counts, size_t max_pairs, int num_sms, cudaStream_t st, int64_t* launches) {
  return zones_of(w, d_levels, n0, n1, n2, axis, n_pairs, sizes, counts, max_pairs, num_sms, st, launches);
}

}  // namespace lm
