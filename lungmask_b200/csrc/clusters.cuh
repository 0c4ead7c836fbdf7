// Size distributions of the 3-D clusters of low-attenuation voxels per label (see clusters.cu, DESIGN §4.7).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kClusterRows = 257;      // rows 1..255 = label values, row 256 = all LAA voxels; row 0 stays empty
constexpr int kClusterDense = 4096;    // cluster sizes below this are counted in a dense [row][size] array

// The pair-count bound of lm_laa_max_pairs: 32 * ceil(sqrt(n)) + 256.
size_t laa_max_pairs(size_t n_voxels);

// Where laa_clusters writes its results (host memory, see lm_laa_clusters_dev in the header).
struct LaaClustersOut {
  int64_t* laa_voxels;   // [257]
  int64_t* n_clusters;   // [257]
  int64_t* n_pairs;      // [257]
  int64_t* sizes;        // [max_pairs]: ascending within a row, rows in order
  int64_t* counts;       // [max_pairs]
  size_t max_pairs;
};

// Device work buffers of laa_clusters, grown on demand and reused across calls.
struct ClusterWork {
  void* d = nullptr;     // parent and area (4 B / voxel each), the two LAA maps (1 B / voxel each), histogram, overflow list
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Clusters of the voxels with mask > 0 and value < threshold in the (n0,n1,n2) volume `d_vol` (element type `dtype`, an
// LM_DTYPE_* code) and the uint8 mask `d_mask`, both on the current device.  conn: 4, 6 or 26.  Enqueues on `st` and
// synchronises it twice (the histogram's extent, then the results).  The caller checks the arguments (n < 2^32,
// max_pairs >= laa_max_pairs(n)).  Returns 0, a cudaError_t, or -1 for an unknown dtype / connectivity.
// *launches += the kernels launched.
int laa_clusters(ClusterWork& w, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2, int threshold,
                 int conn, const LaaClustersOut& out, int num_sms, cudaStream_t st, int64_t* launches);

// The 26-connected equal-value zones of the uint8 (n0,n1,n2) map `d_levels` (0 = outside): n_pairs [256] (row = the map
// value, row 0 zero) and the rows' (size, count) pairs as laa_clusters gives them.  The work area holds parent and area
// (8 B / voxel) and the histogram.  The caller checks the arguments (n < 2^32, max_pairs >= laa_max_pairs(n)).
int zone_sizes(ClusterWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int64_t* n_pairs, int64_t* sizes,
               int64_t* counts, size_t max_pairs, int num_sms, cudaStream_t st, int64_t* launches);

// zone_sizes with 8-connected zones within each plane normal to `axis` (0, 1 or 2).  Axes 1 and 2 permute the map into
// the work area's first map first (1 B / voxel more).  The caller checks the arguments.
int zone_sizes_plane(ClusterWork& w, const uint8_t* d_levels, int n0, int n1, int n2, int axis, int64_t* n_pairs, int64_t* sizes,
                     int64_t* counts, size_t max_pairs, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
