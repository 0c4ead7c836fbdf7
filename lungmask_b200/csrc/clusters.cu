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

// Each labelling has at most n / kClusterDense clusters of kClusterDense voxels or more, and there are two labellings.
size_t over_cap(size_t n) { return 2 * (n / kClusterDense) + 2; }

// Carves the work area; returns its size (d == nullptr: size only).
size_t layout(char* d, size_t n, ClusterDev* g) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = d ? d + off : nullptr; off += align256(bytes); return p; };
  const size_t padded = (n + kChunk - 1) / kChunk * kChunk;
  g->parent = (uint32_t*)take(n * 4);
  g->area = (uint32_t*)take(n * 4);
  g->map_l = (uint8_t*)take(padded);
  g->map_u = (uint8_t*)take(padded);
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
  SC((cudaError_t)w.reserve(layout(nullptr, n, &g)));
  layout(static_cast<char*>(w.d), n, &g);

  SC(cudaMemsetAsync(g.dense, 0, (size_t)kClusterRows * kClusterDense * 4, st));
  SC(cudaMemsetAsync(g.row_max, 0, kClusterRows * 4, st));
  SC(cudaMemsetAsync(g.n_over, 0, 4, st));
  const int rc = map_pass(dtype, d_vol, d_mask, n, threshold, g, num_sms, st);
  if (rc) return rc;
  ++*launches;
  const int g_area = grid_for(cluster_area_kernel, 0, n, num_sms), g_hist = grid_for(cluster_hist_kernel, 0, n, num_sms);
  for (int pass = 0; pass < 2; ++pass) {
    const uint8_t* map = pass ? g.map_u : g.map_l;
    const int lrc = ccl_volume_device(map, g.parent, n0, n1, n2, conn, num_sms, st, launches);
    if (lrc) return lrc;
    SC(cudaMemsetAsync(g.area, 0, n * 4, st));
    cluster_area_kernel<<<g_area, kThreads, 0, st>>>(g.parent, g.area, n);
    cluster_hist_kernel<<<g_hist, kThreads, 0, st>>>(g.parent, g.area, map, n, pass ? 256 : 0, g.dense, g.row_max, g.over, g.n_over);
    SC(cudaGetLastError());
    *launches += 2;
  }

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

}  // namespace lm
