// Device post-processing (see postproc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

// Scratch buffers for postprocess_device, grown on demand and reused across calls.
struct PostScratch {
  size_t cap_vox = 0;
  uint32_t cap_regions = 0;   // region tables hold ids 0..cap_regions (the device flags an overflow, see postprocess_finish)
  uint32_t hash_cap = 0;      // slots of the (area, value) -> lowest id table, a power of two >= 2 * (cap_regions + 1)
  uint32_t sort_cap = 0;      // sort keys, a power of two >= cap_regions
  uint32_t want_regions = 0;  // set by postprocess_finish when a run since the last finish overflowed: capacity the re-run needs
  uint32_t last_regions = 0;  // largest region count seen since the previous postprocess_finish
  bool clear_sticky = true;   // the next run resets the device's sticky overflow flag / region-count maximum
  int ccl_rule = 1;           // 26-connected union-find: 1 = pruned neighbour rule (default), 0 = all 13 backward probes
  int merge_ctas = 0;         // merge loop: 0 = one CTA per SM in batches of independent candidates (cooperative launch),
                              // 1 = the single-CTA sequential loop, n > 1 = that many CTAs
  int debug_stage = 0;        // parity taps: 1 = return the Q5 label map, 2 = region ids & 255, 3 = merged ids & 255
  uint32_t *parent = nullptr, *parent2 = nullptr, *rid = nullptr, *area2 = nullptr;
  uint8_t *mapped = nullptr, *tmp = nullptr, *outside = nullptr;
  uint32_t* block_counts = nullptr;
  uint64_t* small = nullptr;    // 32 KB of small device tables (layout in postproc.cu)
  uint64_t* h_small = nullptr;  // pinned mirror of the first words (R, overflow flag, present labels)
  uint32_t *r_area = nullptr, *r_cur = nullptr, *r_order = nullptr, *r_count = nullptr, *r_touched = nullptr, *r_hslot = nullptr;
  uint8_t *r_value = nullptr, *r_spare_id = nullptr, *r_to_label = nullptr;
  int* r_bbox = nullptr;
  uint64_t *sort_keys = nullptr, *hash_keys = nullptr;
  uint32_t* hash_min = nullptr;
  uint32_t* batch = nullptr;    // multi-CTA merge loop: control words + per-batch member tables
  uint32_t* r_pos = nullptr;    // multi-CTA merge loop: position of every region in the (area, id) order
  int reserve(size_t nvox);
  int reserve_regions(uint32_t R);
  void release();
  void release_regions();
};

// utils.postprocessing on a device-resident (S,H,W) uint8 volume -> d_out (S,H,W) uint8.  Everything is enqueued on
// `st`; with max_label >= 0 (an upper bound of the label values, spare labels included) the call never synchronises
// with the host, otherwise it synchronises ONCE to learn which label values occur.  d_spare (optional) points to
// device ints holding further spare values (n_d_spare of them; the fusion path computes its spare label on device).
// Call postprocess_finish after the stream has been synchronised: it returns 0, or 1 when the region tables
// overflowed (ws.want_regions is set; reserve_regions(want_regions) and run again - the output is invalid).
int postprocess_device(PostScratch& ws, const uint8_t* d_labels, int S, int H, int W, const int32_t* spare, int n_spare,
                       const int32_t* d_spare, int n_d_spare, int skip_below, int max_label, uint8_t* d_out, int num_sms,
                       cudaStream_t st, int64_t* launches, uint32_t* parent_in = nullptr);
int postprocess_finish(PostScratch& ws);
// Slab-wise 3-D labelling (multi-GPU slice sharding): ccl_slab_device labels the slices [z_lo, z_hi) of the (S,H,W) label
// volume on their own into d_parent (global linear indices, neighbours outside the slab ignored; not flattened);
// ccl_join_slabs_device links every slab's first slice (first_slices[0..n_bounds)) to the previous slab and flattens the
// whole volume - the result equals the whole-volume labelling and is what postprocess_device takes as parent_in.
int ccl_slab_device(const uint8_t* d_labels, uint32_t* d_parent, int S, int H, int W, int z_lo, int z_hi, int rule, int num_sms,
                    cudaStream_t st, int64_t* launches);
int ccl_join_slabs_device(const uint8_t* d_labels, uint32_t* d_parent, int S, int H, int W, const int* first_slices, int n_bounds,
                          int num_sms, cudaStream_t st, int64_t* launches);
// Equal-value connected components of a whole (S,H,W) uint8 volume (0 = background) into d_parent: a non-zero voxel gets
// the minimum linear index of its component, a zero voxel 0xFFFFFFFF.  conn: 4 (faces within a slice), 8 (full within a
// slice), 6 (faces) or 26 (full, the default pruned neighbour rule).  Fewer than 2^32 voxels.  Returns 0, a cudaError_t, or -1 for another conn.
int ccl_volume_device(const uint8_t* d_vals, uint32_t* d_parent, int S, int H, int W, int conn, int num_sms, cudaStream_t st,
                      int64_t* launches);
// utils.keep_largest_connected_component on a device-resident (S,H,W) 0/1 mask; -21 if the mask is empty.
int keep_largest_component_device(PostScratch& ws, const uint8_t* d_mask, int S, int H, int W, uint8_t* d_out, int num_sms,
                                  cudaStream_t st);
// utils.reshape_mask for every slice: (S,MH,MW) masks + (S,4) boxes -> (S,H,W).
int reshape_device(const uint8_t* d_masks, const int32_t* d_boxes, int S, int H, int W, int MH, int MW, uint8_t* d_out,
                   int num_sms, cudaStream_t st);
// Per-class probabilities in the native orientation: d_scores (S,K,MH,MW) log-softmax of the LPS volume's slices, boxes
// of those slices -> d_probs (K, n0, n1, n2) float32, p_k = expf(score_k) of the pixel reshape_device samples for the voxel
// (p_0 = 1 where it writes 0).  dims_lps / perm / flip as launch_orient_* (identity perm, no flips: the volume is LPS).
int probs_device(const float* d_scores, const int32_t* d_boxes, int K, int MH, int MW, const int dims_lps[3], const int perm[3],
                 const int flip[3], float* d_probs, int num_sms, cudaStream_t st);
// mask.py:228-230 in place on d_res_l; the spare label value (uint8 arithmetic: max + 1) is left in d_spare_out[0]
// (device int32) for postprocess_device.  No host synchronisation.
int fuse_device(uint8_t* d_res_l, const uint8_t* d_res_r, size_t n, uint32_t* d_scratch, int32_t* d_spare_out, int num_sms,
                cudaStream_t st);
}  // namespace lm
