// Regional statistics support: plane counts, the surface distance transform and region maps (see regions.cu, DESIGN §4.8).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kPlaneRows = 257;   // per plane: columns 0..255 = label values, column 256 = mask > 0

// Device work buffers of the region calls, grown on demand and reused across calls.
struct RegionWork {
  void* d = nullptr;   // distance transform: squared distances (8 B / voxel) and envelope stacks (12 B / voxel);
                       // plane counts [n_axis][257] u64; region map LUT and shell bounds
  size_t d_bytes = 0;
  int reserve(size_t bytes);
  void release();
};

// Voxels per label in every plane along `axis` of the (n0,n1,n2) uint8 mask: counts[p * 257 + l] (host, int64), column
// 256 = mask > 0.  Enqueues on `st` and synchronises it.  The caller checks the arguments.
int plane_label_counts(RegionWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int axis, int64_t* counts, int num_sms,
                       cudaStream_t st, int64_t* launches);

// d_out[v] = float32 of the float64 Euclidean distance from voxel v to the nearest voxel with mask == 0, axis k weighted
// by spacing[k] (0 where mask == 0, +inf without such a voxel; outside the array is not background).  Enqueues on `st`
// (no synchronisation).
int surface_distance(RegionWork& w, const uint8_t* d_mask, int n0, int n1, int n2, const double* spacing, float* d_out,
                     int num_sms, cudaStream_t st, int64_t* launches);

// d_map[v] = lut[bucket(v) * 256 + mask[v]]; bucket = the plane index along `axis` (d_dist == nullptr) or the number of
// the n_bounds float32 `bounds` <= d_dist[v].  lut (host) has n_buckets * 256 entries.  Enqueues on `st` and
// synchronises it (the LUT upload reads host memory).
int region_map(RegionWork& w, const uint8_t* d_mask, const float* d_dist, int n0, int n1, int n2, int axis, const float* bounds,
               int n_bounds, const uint8_t* lut, size_t lut_size, uint8_t* d_map, int num_sms, cudaStream_t st,
               int64_t* launches);

}  // namespace lm
