/* lungmask_b200 — C ABI of the H100-native lungmask hot path.
 *
 * The reference (JoHof/lungmask) is pure Python and has no FFI for this path; the interface each
 * entry point replaces is therefore a Python function of the reference, cited per function
 * (paths relative to the reference root).  The Python shell in lungmask_b200/ binds these with
 * ctypes (INTEGRATION.md shows the stub a maintainer of the reference would add).
 *
 * Conventions: every function returns 0 on success and a non-zero code on failure
 * (lm_last_error() then returns a static, thread-local message); nothing throws.  The caller owns
 * all host buffers; the engine owns all device memory.  One engine drives one CUDA device; calls on
 * one engine must be serialised by the caller.  "dev" variants take device pointers on the engine's
 * device and run on the engine's stream without host copies.
 *
 * Numerics: the convolutions carry every fp32 value as an fp16 pair (hi + lo * 2^-11, 22 significant bits) on the
 * tensor cores and accumulate in fp32; results match the reference's fp32 forward within 1e-4 on the log-softmax
 * scores.  fp16 saturates at 65504: every activation tensor and every layer's weights carry a power-of-two scale
 * (exact: no significand changes); when a value would leave the range the engine lowers that tensor's scale and runs
 * the forward again, transparently.  LM_ERR_RANGE remains only for non-finite weights and for activations beyond
 * about 1e14 - it never returns a silently wrong mask.
 */
#ifndef LUNGMASK_B200_H
#define LUNGMASK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LM_API __attribute__((visibility("default")))
#else
#define LM_API
#endif

typedef struct lm_engine lm_engine;

#define LM_NET_RES 256           /* mask.py:166: utils.preprocess(..., resolution=[256, 256]) */
#define LM_MAX_SLOTS 4           /* weight slots (e.g. 0 = base model, 1 = fill model) */
#define LM_FLAG_NO_POSTPROCESS 1 /* LMInferer(volume_postprocessing=False), mask.py:191-194 */
#define LM_ERR_RANGE (-40)       /* non-finite weight, or an activation beyond every representable scale (see "Numerics") */

/* Engine lifetime.  Replaces LMInferer.__init__'s device pick + model.to(device), mask.py:118-139.
 * batch_capacity = slices per forward wave (the reference's batch_size only bounds memory, results
 * are per-slice independent; mask.py:172-187). */
LM_API int lm_create(int device, int batch_capacity, lm_engine** out);
LM_API void lm_destroy(lm_engine* e);
LM_API const char* lm_last_error(void);
LM_API int lm_device(const lm_engine* e);
LM_API int lm_batch_capacity(const lm_engine* e);

/* Number of floats lm_load_weights expects for a model with n_classes outputs. */
LM_API size_t lm_weight_blob_floats(int n_classes);

/* Replaces get_model()'s load_state_dict + model.to(device), mask.py:54-68.  `blob` is the live
 * tensors of the reference state_dict, fp32, concatenated in this order:
 *   for each of the 18 conv3x3 layers in execution order
 *     (down_path.{0..4}.block.{0,3}, up_path.{0..3}.conv_block.block.{0,3}):
 *       conv.weight (OIHW), conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var
 *   for each up_path.{0..3}.up.1: weight (OI11), bias
 *   last.weight (K,64,1,1), last.bias (K)
 * n_classes = len(last.bias) (mask.py:56). */
LM_API int lm_load_weights(lm_engine* e, int slot, const float* blob, size_t n_floats, int n_classes);

/* LMInferer._inference for numpy input, mask.py:141-210: int16 HU volume (S,H,W) in host memory ->
 * uint8 label volume (S,H,W) in host memory.  flags: LM_FLAG_*. */
LM_API int lm_apply_volume(lm_engine* e, int slot, const int16_t* vol, int S, int H, int W, int flags, uint8_t* out);
/* Same with device-resident input and output (no host<->device copies). */
LM_API int lm_apply_volume_dev(lm_engine* e, int slot, const int16_t* d_vol, int S, int H, int W, int flags, uint8_t* d_out);

/* LMInferer.apply with a fill model, mask.py:223-232 (two inferences + spare-label fusion +
 * postprocessing(spare=[max+1]) at the original resolution).  flags: LM_FLAG_NO_POSTPROCESS reaches the two inner
 * _inference calls only (mask.py:191-194 honours volume_postprocessing there); the fusion post-processing of
 * mask.py:232 is unconditional, exactly as in the reference. */
LM_API int lm_apply_fused(lm_engine* e, int slot_base, int slot_fill, const int16_t* vol, int S, int H, int W, int flags,
                          uint8_t* out);
/* Same with a device-resident input volume and output (no host<->device copies). */
LM_API int lm_apply_fused_dev(lm_engine* e, int slot_base, int slot_fill, const int16_t* d_vol, int S, int H, int W, int flags,
                              uint8_t* d_out);
/* The fusion glue alone, mask.py:228-230: spare = res_l.max() + 1 (uint8 arithmetic); res_l[(res_l == 0) & (res_r > 0)]
 * = spare; res_l[res_r == 0] = 0.  Host (S,H,W) uint8 in, fused (S,H,W) uint8 + the spare value out (parity tap: the
 * array utils.postprocessing(res_l, spare=[spare]) receives at mask.py:232). */
LM_API int lm_fuse(lm_engine* e, const uint8_t* res_l, const uint8_t* res_r, int S, int H, int W, uint8_t* fused,
                   int* spare_value);

/* LMInferer.apply for FLOAT volumes (float32, or float64 with is_f64 != 0), slot_fill >= 0 for the fusion.  The
 * reference keeps the input dtype through utils.preprocess (clip and bilinear zoom without rounding, utils.py:44-45,
 * 108-110) and normalises in that dtype (mask.py:167-168) before the cast to fp32 (mask.py:178-182); so does the engine. */
LM_API int lm_apply_volume_float(lm_engine* e, int slot, int slot_fill, const void* vol, int is_f64, int S, int H, int W,
                                 int flags, uint8_t* out);
/* utils.preprocess(resolution=[256,256]) + the normalisation of mask.py:167-168 for a float volume: the fp32 network
 * input (S,256,256) and the crop boxes (parity tap). */
LM_API int lm_preprocess_float(lm_engine* e, const void* vol, int is_f64, int S, int H, int W, float* normalised,
                               int32_t* boxes);

/* LMInferer.apply for a SimpleITK image, mask.py:157-164,204-208,223-232: the array `vol` (n0,n1,n2) is in the image's
 * NATIVE orientation; lps = transpose(vol, perm) flipped along every axis k with flip[k] != 0 is the array of the image
 * re-oriented to DICOM "LPS" (lungmask_b200/orient.py derives perm / flip from the direction cosines).  The engine
 * re-orients on the device, runs the path on the LPS array and returns the mask in the native orientation (n0,n1,n2).
 * slot_fill >= 0 selects the fusion of mask.py:223-232, whose spare-label fusion and post-processing run on the
 * native-orientation results exactly as in the reference (each _inference call re-orients its own result back). */
LM_API int lm_apply_volume_oriented(lm_engine* e, int slot, int slot_fill, const int16_t* vol, int n0, int n1, int n2,
                                    const int* perm, const int* flip, int flags, uint8_t* out);

/* The mask AND the per-class probabilities of one model, from one forward pass (the reference's `inferer.model(x)`
 * gives the same log-softmax at network resolution).  `vol` (n0,n1,n2) of element type `dtype`: LM_DTYPE_I16 takes the
 * int16 path of lm_apply_volume; LM_DTYPE_F32 / LM_DTYPE_F64 keep their dtype through pre-processing as
 * lm_apply_volume_float does.  perm / flip as lm_apply_volume_oriented; both NULL: the array is already LPS.
 *   out    (n0,n1,n2) uint8: bit-identical to lm_apply_volume / lm_apply_volume_float / lm_apply_volume_oriented with the
 *          same flags (LM_FLAG_NO_POSTPROCESS honoured).
 *   probs  (K,n0,n1,n2) float32 in the native orientation: p_k = expf(s_k), s_k the head's fp32 log-softmax score (the
 *          value lm_forward returns) of the network pixel that the mask's own order-0 resampling (utils.reshape_mask,
 *          utils.py:114-129) places at the voxel.  Voxels that resampling sets to 0 (outside the crop box, or scipy's
 *          constant-mode last row / column) have p_0 = 1 and p_k = 0 for k > 0.  The probabilities are the network's
 *          output BEFORE post-processing, whatever `flags` says; with LM_FLAG_NO_POSTPROCESS argmax_k p_k equals `out`.
 * Device memory: the scores of the whole volume (S * K * 256 * 256 * 4 bytes, S = slices of the LPS volume) and the
 * probabilities (K * n0 * n1 * n2 * 4 bytes) stay allocated in the engine for the next call.  No fusion (slot_fill). */
#define LM_DTYPE_I16 0
#define LM_DTYPE_F32 1
#define LM_DTYPE_F64 2
LM_API int lm_apply_volume_probs(lm_engine* e, int slot, const void* vol, int dtype, int n0, int n1, int n2,
                                 const int* perm, const int* flip, int flags, uint8_t* out, float* probs);

/* The general device-resident entry point: lm_apply_volume / _float / _oriented / _fused / _probs on device memory, for
 * callers that keep their volumes and results on the GPU (a PyTorch pipeline: LMInferer.apply on a CUDA tensor).
 *   d_vol    (n0,n1,n2) C-contiguous on the engine's device, element type `dtype`, in its NATIVE orientation; perm / flip
 *            as lm_apply_volume_oriented, both NULL: the array is LPS.  Never written.  LM_DTYPE_I16 / F32 / F64 take
 *            the paths of the host entry points.  The integer codes (and bool as LM_DTYPE_U8) are clipped to
 *            [-1024, 600] into int16, LM_DTYPE_F16 / BF16 are widened to float32 (LMInferer does the same on the host).
 *   d_out    (n0,n1,n2) uint8 on the device: bit-identical to what the host entry points return for the same volume,
 *            flags and orientation; slot_fill >= 0 selects the fusion (lm_apply_fused / lm_apply_volume_oriented).
 *   d_probs  NULL, or (K,n0,n1,n2) float32 on the device: bit-identical to the probs of lm_apply_volume_probs.  Not with
 *            slot_fill >= 0 (the fusion has no probabilities).
 *   stream   the caller's cudaStream_t (NULL = the legacy default stream).  The engine records an event on it and makes
 *            its own stream wait for that event before it reads d_vol, so work the caller queued on `stream` before the
 *            call (the producer of d_vol) is complete first.  The call returns after the engine stream has
 *            synchronised: d_out and d_probs are complete on return and `stream` needs no further wait.
 * No host<->device copy.  An I16 / F32 / F64 volume in LPS is read in place; any other volume is converted and / or
 * re-oriented into an engine buffer in one pass.  The engine allocates no probability buffer for this call; it keeps
 * its usual work buffers (the whole volume's scores, S * K * 256 * 256 * 4 bytes, when d_probs is given).
 * lm_last_timings: [0] is the wait for `stream` plus the conversion / orientation pass, [5] is the orientation of the
 * results back to the native orientation (with slot_fill >= 0 also the fusion and its post-processing; there is no D2H
 * copy); the other slots as for the host entry points. */
#define LM_DTYPE_U8 3   /* also bool */
#define LM_DTYPE_I8 4
#define LM_DTYPE_I32 5
#define LM_DTYPE_I64 6
#define LM_DTYPE_F16 7
#define LM_DTYPE_BF16 8
LM_API int lm_apply_dev(lm_engine* e, int slot, int slot_fill, const void* d_vol, int dtype, int n0, int n1, int n2,
                        const int* perm, const int* flip, int flags, uint8_t* d_out, float* d_probs, void* stream);

/* Per-label volume and HU statistics of a volume and its label mask (no counterpart in the reference; DESIGN §4.6): what
 * lung-CT tools report from a lungmask result - each lung's or lobe's voxel count, mean / std / min / max HU, percentiles
 * (Perc15) and the fraction of voxels below thresholds (LAA-950).
 *   d_vol    (n0,n1,n2) of element type `dtype` (every LM_DTYPE_* code; bool as LM_DTYPE_U8).  Values are read as they
 *            are: not clipped; float16 / bfloat16 are widened to float32, every value statistic is computed in float64.
 *   d_mask   (n0,n1,n2) uint8, voxel i paired with voxel i of d_vol (orientation does not matter).
 *   percentiles  n_q values q in [0, 100]; thresholds  n_t integers t in [-1024, 3072].
 * Results: 257 rows, row l = the voxels with mask == l (row 0: voxels only), row 256 = the union mask > 0.  NaN values
 * are counted in nan_voxels and excluded from everything else; n = voxels - nan_voxels.
 *   voxels [257], nan_voxels [257]   int64 counts
 *   moments [257][4]       mean, std (population), min, max of the row's values; NaN when n = 0
 *   percentile [257][n_q]  bit-identical to numpy.percentile(values.astype(float64), q) (method "linear"); NaN when n = 0
 *   below_count [257][n_t] count(value < t); 0 when n = 0
 * d_vol and d_mask are device memory of the engine's device; `stream` is the caller's cudaStream_t, with the event-wait
 * rule of lm_apply_dev.  Every argument is checked before any kernel runs; the call returns after the engine's stream has
 * synchronised, and the inputs are never written. */
#define LM_STATS_MAX_PERCENTILES 64
#define LM_STATS_MAX_THRESHOLDS 4097
LM_API int lm_label_stats_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                              const double* percentiles, int n_q, const int* thresholds, int n_t, int64_t* voxels,
                              int64_t* nan_voxels, double* moments, double* percentile, int64_t* below_count, void* stream);

/* Size distributions of the connected clusters of low-attenuation (LAA) voxels per label (no counterpart in the reference;
 * DESIGN §4.7): whether a lobe's LAA-950 is many small holes or a few large bullae (the power-law exponent D of
 * Mishima et al., PNAS 1999, is computed from these pairs by LMInferer.laa_clusters).
 *   d_vol, d_mask as lm_label_stats_dev; a voxel is LAA when mask > 0 and value < threshold, compared in the volume's type
 *                 (integers unclipped, float16 / bfloat16 widened to float32; NaN is never LAA).
 *   threshold     integer HU in [-1024, 3072];  connectivity  4 (faces within a slice, per-slice 2-D clusters), 6 (faces)
 *                 or 26 (full).  Fewer than 2^32 voxels.
 * Results: 257 rows.  Row l (1..255): the components of the LAA voxels with mask == l (a cluster never crosses a label
 * boundary); row 256: the components of all LAA voxels (a cluster may span labels); row 0 is all zero.
 *   laa_voxels [257], n_clusters [257]  int64
 *   n_pairs [257]       the number of distinct cluster sizes of the row
 *   sizes, counts       the (size, count) pairs, ascending by size within a row, rows concatenated in row order
 *                       (sum of n_pairs entries).  max_pairs >= lm_laa_max_pairs(n0*n1*n2), which bounds that sum
 *                       (a row of V LAA voxels has at most sqrt(2V) distinct sizes, the rows hold at most 2n voxels).
 * Device memory, the caller's stream, the argument checks and the return as for lm_label_stats_dev. */
LM_API size_t lm_laa_max_pairs(size_t n_voxels);   /* 32 * ceil(sqrt(n_voxels)) + 256 */
LM_API int lm_laa_clusters_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                               int threshold, int connectivity, int64_t* laa_voxels, int64_t* n_clusters, int64_t* n_pairs,
                               int64_t* sizes, int64_t* counts, size_t max_pairs, void* stream);

/* Regional statistics support (no counterpart in the reference; DESIGN §4.8): craniocaudal zones and depth shells below the
 * lung surface.  LMInferer.regional_statistics turns a zone or shell assignment into a uint8 region map and runs
 * lm_label_stats_dev on it.  All three take device memory of the engine's device and the caller's cudaStream_t with the
 * event-wait rule of lm_apply_dev, check every argument before any kernel runs and return after the engine's stream has
 * synchronised; the inputs are never written.  mask  (n0,n1,n2) uint8.
 * lm_plane_label_counts_dev: the voxels of every label in every plane along array axis `axis` (0, 1 or 2):
 *   counts [n_axis][257] int64 (host), counts[p][l] = the voxels with mask == l in plane p, counts[p][256] = mask > 0.
 * lm_surface_distance_dev: the Euclidean distance in mm from every voxel with mask > 0 to the nearest voxel with
 * mask == 0 (the outside of the union of all labels; fissures between labels are interior), axis k weighted by
 * spacing[k] (3 finite positive doubles, per ARRAY axis).  d_out (n0,n1,n2) float32: the float64 distance rounded once;
 * 0 where mask == 0; +inf when the mask has no zero voxel.  Voxels outside the array are not background (as
 * scipy.ndimage.distance_transform_edt): a lung cut by the first or last slice has no surface there.  Equal to
 * np.float32(scipy.ndimage.distance_transform_edt(mask > 0, sampling=spacing)) bit for bit when every (delta * s_k)^2 and
 * their sums are exact in float64 (dyadic spacings such as 0.703125 or 1.25), else within 1 float32 ulp.  Work area:
 * 20 bytes per voxel, kept by the engine.
 * lm_region_map_dev: d_map[v] = lut[bucket(v) * 256 + mask[v]] (n0,n1,n2 uint8).  d_dist NULL: bucket = the plane index
 * of v along `axis` (0, 1 or 2), n_bounds 0, n_axis buckets.  Otherwise bucket = the number of the n_bounds float32
 * `bounds` (finite, positive, strictly increasing, at most 254; host memory) that are <= d_dist[v] (float32 (n0,n1,n2),
 * e.g. from lm_surface_distance_dev), n_bounds + 1 buckets; `axis` is ignored.  lut (host): buckets * 256 codes
 * (lut_size), lut[b * 256 + 0] == 0 for every b. */
LM_API int lm_plane_label_counts_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int axis, int64_t* counts,
                                     void* stream);
LM_API int lm_surface_distance_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, const double* spacing,
                                   float* d_out, void* stream);
LM_API int lm_region_map_dev(lm_engine* e, const uint8_t* d_mask, const float* d_dist, int n0, int n1, int n2, int axis,
                             const float* bounds, int n_bounds, const uint8_t* lut, size_t lut_size, uint8_t* d_map,
                             void* stream);

/* ---- one volume over several GPUs (SURVEY.md 8e; the reference is single-device, mask.py:118-121) ----------------
 * One process and one engine per GPU.  Slices are independent up to the 3-D post-processing (utils.py:48-51,
 * mask.py:173-187,196-202 vs utils.py:293-358): rank r of `world` runs pre-processing and the network on the contiguous
 * slice range [r * ceil(S/world), (r+1) * ceil(S/world)) and the uint8 argmax volume (plus the crop boxes) is
 * all-gathered once - by the engine itself: every rank owns a gather block in device memory that its peers map through
 * CUDA IPC, a rank pushes its slab into every peer's block over NVLink and raises an epoch flag there; post-processing
 * and reshape then run replicated on the gathered volume and every rank holds the whole result.  The 3-D labelling of
 * utils.py:293 is slab-sharded too: every rank labels its own slices, the union-find parents travel with the labels,
 * and after the gather only the slab boundaries are linked ("shard_slab_ccl", default 1).
 *   lm_shard_init     allocates this rank's gather block for volumes of up to max_slices slices
 *   lm_shard_export   writes the block's IPC handle (lm_shard_handle_bytes() bytes) - exchange it by any host channel
 *   lm_shard_connect  maps the peers' blocks; `handles` = world handles in rank order (this rank's own is ignored)
 *   lm_apply_volume_sharded      every rank passes the SAME (S,H,W) host volume (only its slab is copied to the device)
 *                                and receives the whole (S,H,W) result (out may be NULL on ranks that do not need it)
 *   lm_apply_volume_sharded_dev  device-resident whole-volume buffers on this rank's device (only the slab is read)
 *   lm_shard_labels   parity / alternative-collective tap: device pointers of this rank's gathered boxes (int32 x 4
 *                     per slice) and labels (256*256 bytes per slice), and the slice capacity
 * The calls are collective: every rank must make them in the same order (a bounded device-side wait turns a missing
 * peer into error -50 instead of a hang).  world == 1 needs no export / connect. */
LM_API int lm_shard_init(lm_engine* e, int rank, int world, int max_slices);
LM_API size_t lm_shard_handle_bytes(void);
LM_API int lm_shard_export(lm_engine* e, void* handle_out);
LM_API int lm_shard_connect(lm_engine* e, const void* handles);
LM_API int lm_shard_labels(lm_engine* e, void** d_boxes, void** d_labels, size_t* slice_cap);
LM_API int lm_apply_volume_sharded(lm_engine* e, int slot, const int16_t* vol, int S, int H, int W, int flags, uint8_t* out);
LM_API int lm_apply_volume_sharded_dev(lm_engine* e, int slot, const int16_t* d_vol, int S, int H, int W, int flags,
                                       uint8_t* d_out);

/* ---- stage-level entry points (each mirrors one reference function; used by the parity tests) ---- */

/* utils.preprocess(img, resolution=[out_h,out_w]), utils.py:32-52 (+ simple_bodymask :55-82,
 * crop_and_resize :85-111): (S,H,W) int16 -> resized (S,out_h,out_w) int16 + boxes (S,4) int32
 * [r0, c0, r1, c1] half-open.  clip != 0 applies np.clip(-1024, 600) (utils.py:45) as preprocess does;
 * clip == 0 gives utils.crop_and_resize on each slice as-is. */
LM_API int lm_preprocess(lm_engine* e, const int16_t* vol, int S, int H, int W, int out_h, int out_w, int clip,
                         int16_t* resized, int32_t* boxes);
/* utils.simple_bodymask, utils.py:55-82: one slice (H,W) int16 (NOT clipped) -> (H,W) uint8 0/1. */
LM_API int lm_simple_bodymask(lm_engine* e, const int16_t* slice, int H, int W, uint8_t* mask);

/* Normalise + UNet.forward + argmax, mask.py:167-187 / resunet.py:58-70: resized (S,256,256) int16 ->
 * labels (S,256,256) uint8 and, if scores != NULL, the LogSoftmax scores (S,K,256,256) fp32. */
LM_API int lm_forward(lm_engine* e, int slot, const int16_t* resized, int S, uint8_t* labels, float* scores);

/* utils.postprocessing(label_image, spare, skip_below), utils.py:272-358 on a (S,H,W) uint8 volume. */
LM_API int lm_postprocess(lm_engine* e, const uint8_t* labels, int S, int H, int W, const int32_t* spare, int n_spare,
                   int skip_below, uint8_t* out);

/* utils.keep_largest_connected_component(mask), utils.py:390-404: (S,H,W) uint8 0/1 mask -> 0/1 mask of its largest
 * full-connectivity component (ties: the last in raster order).  Fails (like the reference) on an empty mask. */
LM_API int lm_keep_largest_component(lm_engine* e, const uint8_t* mask, int S, int H, int W, uint8_t* out);

/* [utils.reshape_mask(mask[i], boxes[i], (H,W)) for i], utils.py:114-129 + mask.py:196-202:
 * (S,mask_h,mask_w) uint8 + boxes -> (S,H,W) uint8. */
LM_API int lm_reshape_masks(lm_engine* e, const uint8_t* masks, int mask_h, int mask_w, const int32_t* boxes, int S,
                            int H, int W, uint8_t* out);

/* Per-stage device time (ms, CUDA events on the engine stream) of the last lm_apply_volume* / lm_apply_dev:
 * [0] H2D, [1] preprocess, [2] forward, [3] postprocess, [4] reshape, [5] D2H, [6] total (lm_apply_dev: see there).
 * Also the number of kernels the engine launched in that call. */
LM_API int lm_last_timings(const lm_engine* e, float* ms7, int64_t* kernel_launches);

/* Options: "time_convs" (0/1: bracket every tensor-core convolution launch with CUDA events on the engine
 * stream; read the sum with lm_last_conv_timing after an lm_apply_volume* call), "chunk_kb" (k-blocks
 * accumulated inside the tensor core between fp32 round-to-nearest adds; sets both layer classes),
 * "chunk_kb_wide" (the same for the layers with >= 128 output channels only; defaults: 1 for the 64-channel
 * layers, 2 for the wide ones), "weight_mcast" (0 / 2: clusters of two CTAs share every weight stage through TMA
 * multicast; bit-identical, default 0),
 * "conv64_cm" (1, default: the three 3x3 layers with 64 output channels at full resolution run as channel-major
 * 16x16-pixel tiles, conv_cm64_kernel; 0: the BN = 64 kernel; bit-identical; environment LM_CONV64_CM at lm_create),
 * "stem_v2" (0 = first stem kernel, 1 = register-resident, 2 = shared-memory tile, 3 = the same with the next tile's
 * samples fetched one tile ahead, the default; all bit-identical),
 * "graphs" (1, default: a volume's forward - every wave's ~26 launches - is captured once as a CUDA graph and replayed;
 * 0: every kernel is launched individually; per-launch convolution timing and score taps always launch individually),
 * "upsample_v2" (0: one thread per output sample, 1: per cell, 2 = default: per cell with static corner indexing; all bit-identical),
 * "merge_ctas" (0, default: the region merge loop of utils.py:310-339 runs on one CTA per SM in batches of independent
 * candidates; 1: the single-CTA sequential loop; n: that many CTAs),
 * "ccl_rule" (1 = pruned neighbour rule of the 26-connected labelling, the default; 0 = probe all 13 backward
 * neighbours), "post_region_capacity" (test hook: size of the post-processing's region tables),
 * "post_debug_stage" (parity taps of the post-processing). */
LM_API int lm_set_option(lm_engine* e, const char* key, int value);
LM_API int lm_last_conv_timing(const lm_engine* e, float* conv_ms, int64_t* conv_launches);

/* Parity taps: intermediate activations of the LAST forward wave, as fp32 [n][H][W][C] (channels last; the
 * hi/lo operand planes are joined).  Activation ids follow the execution order of the network:
 * 0 A0(stem out) 1 S0 2 P0 3 A1 4 S1 5 P1 6 A2 7 S2 8 P2 9 A3 10 S3 11 P3 12 A4 13 B4 (encoder: A = first conv,
 * S = block output / skip, P = pooled) 14 L0 15 U0 16 C0 17 E0 18 L1 19 U1 20 C1 21 E1 22 L2 23 U2 24 C2 25 E2
 * 26 L3 27 U3 28 C3 (decoder: L = 1x1 conv below the upsample, U = upsampled, C = first conv, E = block output). */
LM_API int lm_debug_activation_info(int act_id, int* level, int* channels, int* split);
LM_API int lm_debug_read_activation(lm_engine* e, int act_id, int n, float* out);

/* Forward-only benchmark hook: runs the forward pass on `S` device-resident resized slices and
 * reports the device time of the convolution kernels alone (ms) for the roofline. */
LM_API int lm_forward_dev(lm_engine* e, int slot, const int16_t* d_resized, int S, uint8_t* d_labels, float* conv_ms);

#ifdef __cplusplus
}
#endif
#endif /* LUNGMASK_B200_H */
