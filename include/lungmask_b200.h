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

/* Grey-level texture matrices of one ROI (no counterpart in the reference; DESIGN §4.9): LMInferer.texture computes the
 * GLCM, GLSZM, GLRLM, GLDM and NGTDM features of every row of lm_label_stats_dev from these.  All take device memory of the engine's
 * device and the caller's cudaStream_t with the event-wait rule of lm_apply_dev, check every argument before any kernel
 * runs and return after the engine's stream has synchronised; the inputs are never written.  Fewer than 2^32 voxels.
 * lm_texture_levels_dev: the uint8 level map of one row.  d_vol, dtype, d_mask as lm_label_stats_dev; row 1..255 (the
 *   voxels with mask == row) or 256 (mask > 0).  The ROI is the row's voxels with a non-NaN value (float16 / bfloat16
 *   widened to float32); there d_levels[v] = floor((floor(x) - low) / bin_width) + 1, computed in int64, and 0
 *   elsewhere.  bin_width >= 1, n_levels 1..255.  d_levels: n0*n1*n2 bytes, 16-byte aligned.  A level outside
 *   1..n_levels or a non-finite value in the ROI is an error (the map is then incomplete).
 * lm_glcm_dev: the unordered pair counts of a level map (0 = outside the ROI) with levels 1..n_levels (a larger level is
 *   an error).  For each of the 13 offsets d of the 26-neighbourhood whose first non-zero component is positive, in the
 *   order (0,0,1), (0,1,-1), (0,1,0), (0,1,1), then (1,dy,dx) for dy, dx = -1, 0, 1 (array axes 0, 1, 2), U_d(i, j),
 *   i <= j, is the number of voxel pairs (v, v + d) inside the array with levels {i, j}.  counts (host): int64
 *   [13][n_levels (n_levels + 1) / 2], (i, j) in row-major upper-triangle order (i = 1: j = 1..n_levels, then i = 2 ...).
 * lm_zone_sizes_dev: the 26-connected components of equal level of a level map (0 = outside): n_pairs [256] int64 (row =
 *   level; row 0 is 0), sizes and counts as lm_laa_clusters_dev (ascending sizes within a row, rows in order),
 *   max_pairs >= lm_laa_max_pairs(n0*n1*n2).
 * lm_glrlm_dev: the run counts of a level map with levels 1..n_levels (a larger level is an error).  For each of the 13
 *   offsets d of lm_glcm_dev, in its order, a run is a maximal sequence v, v+d, ..., v+(k-1)d of voxels inside the array
 *   that all have level i >= 1.  counts (host): int64 [13][n_levels][max(n0,n1,n2)], the runs of level i+1 and length
 *   k+1 along direction d.
 * lm_neighbour_counts_dev: for each voxel v of level i >= 1 (levels 1..n_levels as lm_glrlm_dev), W(v) is the number of
 *   its 26 neighbours inside the array with level >= 1, S(v) the sum of their levels, and c(v) the number of those with
 *   |level - i| <= alpha (alpha >= 0).  dependence, ngtdm_counts, ngtdm_sums (host): int64 [n_levels][27], G(i, c) the
 *   voxels of level i with c(v) = c, N(i, W) those with W(v) = W, A(i, W) = the sum of |W i - S(v)| over them. */
LM_API int lm_texture_levels_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                                 int row, int64_t low, int bin_width, int n_levels, uint8_t* d_levels, void* stream);
LM_API int lm_glcm_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts,
                       void* stream);
LM_API int lm_zone_sizes_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int64_t* n_pairs, int64_t* sizes,
                             int64_t* counts, size_t max_pairs, void* stream);
LM_API int lm_glrlm_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts,
                        void* stream);
LM_API int lm_neighbour_counts_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                                   int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums, void* stream);

/* Texture matrices over generalised neighbourhoods (DESIGN §4.18): PyRadiomics' distances and force2D settings, for
 * LMInferer.texture.  Device memory, stream rule, checks, synchronisation and levels as for lm_glcm_dev.
 * offsets (host): int8 [n_offsets][3] (dz, dy, dx) over array axes (0, 1, 2), 1 <= n_offsets <= 171, each with
 *   components in -3..3, Chebyshev norm >= 1 and a positive first non-zero component, no two equal.
 * lm_glcm_offsets_dev: U_o(i <= j) as lm_glcm_dev for each offset o in the given order: counts int64 [n_offsets][T].
 * lm_neighbour_offsets_dev: lm_neighbour_counts_dev over the K = 2 n_offsets neighbours v +- o: dependence,
 *   ngtdm_counts, ngtdm_sums int64 [n_levels][K + 1].
 * lm_zone_sizes_plane_dev: lm_zone_sizes_dev with zones 8-connected within each plane normal to `axis` (0, 1 or 2). */
LM_API int lm_glcm_offsets_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels,
                               const int8_t* offsets, int n_offsets, int64_t* counts, void* stream);
LM_API int lm_neighbour_offsets_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                                    const int8_t* offsets, int n_offsets, int64_t* dependence, int64_t* ngtdm_counts,
                                    int64_t* ngtdm_sums, void* stream);
LM_API int lm_zone_sizes_plane_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int axis, int64_t* n_pairs,
                                   int64_t* sizes, int64_t* counts, size_t max_pairs, void* stream);

/* Mesh shape support (no counterpart in the reference; DESIGN §4.10): LMInferer.shape computes PyRadiomics-style shape
 * features (surface area, mesh volume, sphericity, maximum diameters, principal axes) of every row of lm_label_stats_dev
 * from these.  Both take device memory of the engine's device and the caller's cudaStream_t with the event-wait rule of
 * lm_apply_dev, check every argument before any kernel runs and return after the engine's stream has synchronised; the
 * mask is never written.  mask (n0,n1,n2) uint8, fewer than 2^32 voxels and every axis below 2^30.  A voxel is in row l
 * (1..255) when mask == l and in row 256 when mask != 0; voxels outside the array are in no row (the mask is padded with
 * one voxel of outside, the opposite of lm_surface_distance_dev).  A cube is each 2x2x2 block of the padded grid, with
 * lowest corner p (p_k in -1..n_k-1); its configuration has bit c set when corner p + ((c >> 2) & 1, (c >> 1) & 1, c & 1)
 * is in the row.
 * lm_shape_sums_dev: one pass for all rows (host int64 results; row 0 stays zero):
 *   cube_counts [257][256]     the cubes of each configuration (0 and 255 stay zero)
 *   cube_possum [257][256][3]  the sum of their lowest corners p over the array axes
 *   moments [257][10]          N, sum i, sum j, sum k, sum i^2, sum j^2, sum k^2, sum ij, sum ik, sum jk over the row's
 *                              voxels (i, j, k) in array axes
 * lm_max_diameters_dev: d2 [4] (host doubles), the largest squared distance (mm^2) between two mesh vertices of `row`
 *   (1..256) - all pairs, pairs with equal axis-0, equal axis-1 and equal axis-2 coordinate.  A vertex is the midpoint
 *   u + v (doubled integer coordinates) of two face-adjacent grid points of the padded grid that differ in membership;
 *   d^2 = ((D2 h2)^2 + (D1 h1)^2) + (D0 h0)^2 with h_k = spacing[k] / 2 (spacing per ARRAY axis, finite and positive),
 *   every product and sum rounded on its own; 0 without a pair.  Work area: 8 bytes per line of the grid along each axis
 *   and edge direction, and 16 bytes per candidate vertex, kept by the engine. */
LM_API int lm_shape_sums_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int64_t* cube_counts,
                             int64_t* cube_possum, int64_t* moments, void* stream);
LM_API int lm_max_diameters_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const double* spacing,
                                double* d2, void* stream);

/* Surface meshes (no counterpart in the reference; DESIGN §4.14): the marching-cubes mesh of one row that
 * lm_shape_sums_dev's SurfaceArea and MeshVolume describe, so that LMInferer.mesh can return it and io.save_mesh write it
 * as STL, OBJ or PLY.  Both take device memory of the engine's device and the caller's cudaStream_t with the event-wait
 * rule of lm_apply_dev, check every argument before any kernel runs and return after the engine's stream has
 * synchronised; the mask is never written.  mask (n0,n1,n2) uint8 and row (1..256) as lm_max_diameters_dev, on the mask
 * padded with one voxel of outside (grid points q with q_k in -1..n_k).
 *   Vertices: one per crossing edge, the edge from grid point q to q + e_m (m = 0, 1, 2 an array axis) whose ends differ
 *   in membership; ordered by q in the padded grid's linear order (axis 0 slowest), then m.
 *   Triangles: each cube (lowest corner p) gets the triangles of its configuration from the caller's table, ordered by
 *   cube in the padded linear order, then table order.  tri_offsets [257] (host int32, non-decreasing from 0, at most
 *   16 triangles per configuration, none for configurations 0 and 255): configuration c owns triangles
 *   [tri_offsets[c], tri_offsets[c + 1]); tri_codes [3 tri_offsets[256]] (host uint8): per triangle vertex the code
 *   (a << 2) | m of the cube edge from corner a (0..7, as lm_shape_sums_dev numbers them, with bit 2 - m clear) to corner
 *   a + e_m, which must cross in that configuration.  The edge names the vertex owned by (p + corner a, m).
 * lm_mesh_counts_dev: *n_vertices = V, *n_triangles = T (host int64).
 * lm_mesh_emit_dev: n_vertices and n_triangles must equal V and T (the call recounts them), each at most 2^31 - 1.
 *   d_index2 (V,3) int32: the doubled array-axis coordinates 2q + e_m of every vertex (exact).
 *   d_vertices (V,3) float64: with (x, y, z) = (u2, u1, u0) / 2 of u = index2, o = geometry[0..2] (mm), D = geometry[3..11]
 *     (row-major 3x3, columns = array axes 2, 1, 0) and s = geometry[12..14] (spacing x, y, z in mm, positive), p_c =
 *     ((o_c + D[c][0] (s_x x)) + D[c][1] (s_y y)) + D[c][2] (s_z z), every product and sum rounded on its own (no fused
 *     multiply-add); LM_MESH_RAS negates p_0 and p_1.
 *   d_triangles (T,3) int32: vertex indices; the last two are swapped when det D < 0, so that the normals point out of
 *     the row in patient space as the table's do in (x, y, z).
 *   Work area: the table and 16 bytes per line of the padded grid along axis 2 ((n0 + 1) (n1 + 1) lines), kept by the
 *   engine. */
#define LM_MESH_RAS 1
LM_API int lm_mesh_counts_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const int32_t* tri_offsets,
                              const uint8_t* tri_codes, int64_t* n_vertices, int64_t* n_triangles, void* stream);
LM_API int lm_mesh_emit_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const int32_t* tri_offsets,
                            const uint8_t* tri_codes, const double* geometry, int flags, int64_t n_vertices,
                            int64_t n_triangles, int32_t* d_index2, double* d_vertices, int32_t* d_triangles, void* stream);

/* First-order (histogram) sums (no counterpart in the reference; DESIGN §4.11): LMInferer.first_order computes
 * PyRadiomics' 18 default firstorder features of every row of lm_label_stats_dev from these two passes.  Both take
 * device memory of the engine's device and the caller's cudaStream_t with the event-wait rule of lm_apply_dev, check
 * every argument before any kernel runs and return after the engine's stream has synchronised; the inputs are never
 * written.  d_vol, dtype, d_mask as lm_label_stats_dev, fewer than 2^32 voxels.  A voxel is in row l (1..255) when
 * mask == l and in row 256 when mask > 0; a row's ROI is its voxels with a non-NaN value (float16 / bfloat16 widened to
 * float32, every value read as float64).
 * Row inputs (host arrays indexed 0..256, row 0 unused): mode 0 (skip), 1 (float) or 2 (exact: integer volumes only);
 *   a label row with a mode needs row 256 with one.  band_lo <= band_hi: the band, compared in float64, both inclusive.
 *   base: an exact row's integer minimum (|base| <= 2^53); its values must lie in [base, base + 2^20).  centre: a float
 *   row's finite centre.
 * lm_first_order_sums_dev (pass A): level = floor((floor(x) - low) / bin_width) + 1 in int64 as lm_texture_levels_dev,
 *   which must lie in 1..n_levels (1..255).  Host results, zero for skipped rows:
 *   histogram [257][256] int64    the ROI's voxels per level (index 0 unused)
 *   int_sums [257][10] uint64     exact rows: S1, S2, S3, S4, S_B as 128-bit (low word, high word) pairs, S_k = sum d^k
 *                                 with d = x - base, S_B = sum d over the band
 *   band_count [257] int64        the ROI's voxels in the band
 *   float_sums [257][5] float64   float rows: sum e, e^2, e^3, e^4 with e = x - centre, and sum e over the band
 * lm_first_order_splits_dev (pass B).  Host results, zero for skipped rows:
 *   below [257][4] int64          exact rows: the count and the sum of d of the ROI's voxels with d <= split, then of the
 *                                 band's voxels with d <= split_band (split, split_band in [0, 2^20))
 *   abs_dev [257][2] float64      float rows: sum |x - centre| over the ROI, sum |x - centre_band| over the band
 * The integer results are exact and independent of the schedule; the float sums are order-dependent in the last bits.
 * A value of an exact row outside its span or a level outside 1..n_levels is an error.  Work area: a row table, a
 * 2 KB histogram and 88 bytes of sums per row, kept by the engine. */
LM_API int lm_first_order_sums_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                                   int bin_width, const int* mode, const int64_t* low, const int* n_levels,
                                   const int64_t* base, const double* centre, const double* band_lo, const double* band_hi,
                                   int64_t* histogram, uint64_t* int_sums, int64_t* band_count, double* float_sums,
                                   void* stream);
LM_API int lm_first_order_splits_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1,
                                     int n2, const int* mode, const int64_t* base, const int64_t* split,
                                     const int64_t* split_band, const double* centre, const double* centre_band,
                                     const double* band_lo, const double* band_hi, int64_t* below, double* abs_dev,
                                     void* stream);

/* Wavelet decomposition (no counterpart in the reference; DESIGN §4.12): one band of PyRadiomics' getWaveletImage with
 * its defaults (pywt.swtn, level 1, start_level 0), so that LMInferer.wavelet_features can run the first-order and
 * texture calls on every decomposition.
 * lm_wavelet_dev writes band `band` (0..7 = 4 h_x + 2 h_y + h_z, h = 1 for the high-pass filter along that axis:
 *   1 LLH, 2 LHL, 3 LHH, 4 HLL, 5 HLH, 6 HHL, 7 HHH, 0 LLL) of the (n0,n1,n2) volume d_vol (every LM_DTYPE_* code; bool
 *   as LM_DTYPE_U8; converted to float64 first) to the float64 (n0,n1,n2) d_out.  The passes run along array axis 2 (x),
 *   then 1 (y), then 0 (z): out[o] = sum_{j=0..F-1} f[j] in[(o + F/2 - j) mod N'], summed from +0.0 with j ascending, each
 *   product and each sum rounded to float64 with no fused multiply-add; an odd axis of N voxels is wrapped to
 *   N' = N + 1 (index N holds index 0) and the result trimmed back to N.  Filters: PyWavelets' dec_lo of `wavelet` and
 *   dec_hi[k] = (-1)^(k+1) dec_lo[F-1-k]; coif1 (F = 6) or haar (F = 2).  Every padded extent N' must be at least F and
 *   the volume must hold fewer than 2^32 voxels; d_out must not overlap d_vol.  Device memory of the engine's device, the
 *   caller's cudaStream_t with the event-wait rule of lm_apply_dev; every argument is checked before any kernel runs and
 *   the call returns after the engine's stream has synchronised.  A NaN or +-inf anywhere in the volume returns
 *   LM_ERR_NONFINITE (d_out is then not a band).  Work area: one flag; no full-volume intermediate. */
#define LM_WAVELET_COIF1 0
#define LM_WAVELET_HAAR 1
#define LM_ERR_NONFINITE (-41)   /* lm_wavelet_dev: the volume holds a NaN or +-inf */
LM_API int lm_wavelet_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, int wavelet, int band,
                          double* d_out, void* stream);

/* Image filters (no counterpart in the reference; DESIGN §4.13): PyRadiomics' Square, SquareRoot, Logarithm, Exponential
 * and Gradient image types with their defaults, so that LMInferer.filtered_features can run the first-order and texture
 * calls on them.  All three calls take the (n0,n1,n2) volume d_vol (every LM_DTYPE_* code; bool as LM_DTYPE_U8; each
 * voxel converted to float64), fewer than 2^32 voxels, device memory of the engine's device and the caller's
 * cudaStream_t with the event-wait rule of lm_apply_dev; every argument is checked before any kernel runs, the call
 * returns after the engine's stream has synchronised, and a NaN or +-inf anywhere in the volume returns
 * LM_ERR_NONFINITE (the outputs are then not an image).  Work area: a flag and 24 KB of range partials.
 * lm_image_range_dev writes the volume's min and max (as float64) to the host out[2].
 * lm_image_filter_dev writes image type `type` (LM_FILTER_*) to the float64 (n0,n1,n2) d_out, which must not overlap
 *   d_vol or the table.  With d_table NULL it computes, with c = params[0] formed by the caller in float64 from
 *   m = max|x|: SQUARE t = c x, t t (c = 1/sqrt(m)); SQUAREROOT x > 0: sqrt(x c), x < 0: -sqrt(-x c), else x (c = m);
 *   LOGARITHM x > 0: log(x + 1), x < 0: -log(-(x - 1)), else x, then times c (c = m / log(m + 1)); EXPONENTIAL
 *   exp(c x) (c = log(m) / m); each product, sum and square root rounded to float64 with no fused multiply-add, log and
 *   exp CUDA's (within 1 ulp).  With d_table (integer dtypes only; device float64 [table_len], 1 <= table_len <= 2^20)
 *   it writes d_table[x - table_min]; a voxel outside [table_min, table_min + table_len) returns LM_ERR_TABLE_RANGE.
 * lm_gradient_dev writes ITK's GradientMagnitudeImageFilter to the float64 (n0,n1,n2) d_out (not overlapping d_vol):
 *   per axis i (x = array axis 2, y = 1, z = 0) g_i = ((0 + k0 f[-1]) + k1 f[0]) + k2 f[+1] with (k0, k1, k2) =
 *   (-0.5, 0, 0.5) * (1.0 / spacing_xyz[i]) and neighbours outside the array clamped to the edge voxel, then
 *   sqrt(((0 + g_x^2) + g_y^2) + g_z^2), each product, sum and the square root rounded to float64.  spacing_xyz: 3
 *   finite positive sizes in mm (x, y, z). */
#define LM_FILTER_SQUARE 0
#define LM_FILTER_SQUAREROOT 1
#define LM_FILTER_LOGARITHM 2
#define LM_FILTER_EXPONENTIAL 3
#define LM_ERR_TABLE_RANGE (-42)   /* lm_image_filter_dev: a voxel lies outside the table */
LM_API int lm_image_range_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, double* out,
                              void* stream);
LM_API int lm_image_filter_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, int type,
                               const double* params, const double* d_table, int64_t table_min, int64_t table_len,
                               double* d_out, void* stream);
LM_API int lm_gradient_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, const double* spacing_xyz,
                           double* d_out, void* stream);

/* Resampling (no counterpart in the reference; DESIGN §4.19): PyRadiomics' resampleImage with the sitkBSpline or
 * sitkNearestNeighbor interpolator, for LMInferer.resample.  Both calls take the (n0,n1,n2) volume d_vol (every
 * LM_DTYPE_* code; bool as LM_DTYPE_U8), fewer than 2^32 voxels, device memory of the engine's device and the caller's
 * cudaStream_t with the event-wait rule of lm_apply_dev; every argument is checked before any kernel runs and the call
 * returns after the engine's stream has synchronised.  Work area: one flag.
 * lm_bspline_coefficients_dev writes the cubic B-spline coefficients (mirror boundaries, pole z = sqrt(3) - 2) of the
 *   volume, converted to float64, to the float64 (n0,n1,n2) d_coeff (not overlapping d_vol): the 1-D decomposition along
 *   array axis 2 (x), then 1 (y), then 0 (z); per line of N > 1 samples: times (1 - z)(1 - 1/z); c[0] = c[0] +
 *   sum_{n=1..17} z^n c[n] (N >= 19) or Thevenaz's full mirror sum (N <= 18, z^(N-1) formed by repeated products);
 *   c[n] += z c[n-1]; c[N-1] = (z / (z z - 1)) (z c[N-2] + c[N-1]); c[n] = z (c[n+1] - c[n]); each product, sum and the
 *   one division rounded to float64 on its own, with no fused multiply-add.  A NaN or +-inf anywhere in the volume
 *   returns LM_ERR_NONFINITE (d_coeff is then not the coefficients).
 * lm_resample_dev samples the volume at the (m0,m1,m2) points (d_cz[k0], d_cy[k1], d_cx[k2]) of the input's continuous
 *   index (device float64 tables [m0], [m1], [m2], finite, fewer than 2^32 points): a point with c < -0.5 or
 *   c >= N - 0.5 along any axis gets 0 in d_out and d_out_mask.  d_out_mask (m0,m1,m2) uint8 gets the uint8 (n0,n1,n2)
 *   d_mask at floor(c + 0.5) of each axis (clamped to [0, N - 1]); d_out (m0,m1,m2) of `dtype` gets, under
 *   LM_RESAMPLE_NEAREST, d_vol at that voxel, and under LM_RESAMPLE_BSPLINE the cubic B-spline of d_coeff (the output of
 *   lm_bspline_coefficients_dev for d_vol): per axis w = c - floor(c), w3 = w^3 / 6, w0 = 1/6 + w (w - 1) / 2 - w3,
 *   w2 = w + w0 - 2 w3, w1 = 1 - w0 - w2 - w3 on the indices floor(c) - 1 .. floor(c) + 2 mirrored with period 2N - 2
 *   (0 when N = 1), the 64 taps summed x innermost, then y, then z, each sum from +0.0, rounded as above.  The value is
 *   stored in `dtype`: integers clamped to the type's range (int64: to 2^63 - 1024) and truncated toward zero, float32 and
 *   float16 rounded to nearest, bfloat16 rounded to float32 and then to bfloat16, float64 kept.  d_coeff is not read
 *   (and may be NULL) under LM_RESAMPLE_NEAREST.  The outputs must not overlap each other or any input.  A sampled value
 *   that is a NaN or +-inf returns LM_ERR_NONFINITE. */
#define LM_RESAMPLE_BSPLINE 0
#define LM_RESAMPLE_NEAREST 1
LM_API int lm_bspline_coefficients_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, double* d_coeff,
                                       void* stream);
LM_API int lm_resample_dev(lm_engine* e, const void* d_vol, int dtype, const double* d_coeff, const uint8_t* d_mask, int n0,
                           int n1, int n2, const double* d_cz, const double* d_cy, const double* d_cx, int m0, int m1,
                           int m2, int interpolator, void* d_out, uint8_t* d_out_mask, void* stream);

/* Laplacian of Gaussian (no counterpart in the reference; DESIGN §4.20): PyRadiomics' LoG image type, ITK's
 * LaplacianRecursiveGaussianImageFilter with NormalizeAcrossScale, for LMInferer.log_images.  The (n0,n1,n2) volume d_vol
 * (every LM_DTYPE_* code; bool as LM_DTYPE_U8; converted to float64), every extent >= 4 and fewer than 2^32 voxels, device
 * memory of the engine's device and the caller's cudaStream_t with the event-wait rule of lm_apply_dev; every argument
 * is checked before any kernel runs and the call returns after the engine's stream has synchronised.  Work area: one
 * flag, and the caller's d_work0 and d_work1, float64 (n0,n1,n2) volumes.
 * spacing_xyz: 3 finite positive sizes in mm (x = array axis 2, y = 1, z = 0); sigma_mm finite and > 0, with every axis
 * d holding at least ceil(sigma_mm / spacing_xyz[d]) + 1 voxels.  The engine forms the coefficients itself, per axis
 * with sd = sigma_mm / spacing_xyz[d], by the float64 operations of lungmask_b200.laplacian.coefficients in the same
 * order (libm sin, cos and exp; Deriche's constants; order 0 normalised to unit sum, order 2 to sd^2 times the second
 * derivative).  d_out (n0,n1,n2) float64 gets, for d = x, y, z, the order-0 line filter along the two other axes in
 * x, y, z order and then the order-2 line filter along d, the three terms summed from +0.0 in that order.  A line filter
 * is the causal and anticausal 4th-order recursion of ITK's RecursiveSeparableImageFilter, the taps outside the line
 * reading the end sample (rows in lungmask_b200/laplacian.py), every product and sum rounded to float64 on its own with
 * no fused multiply-add: d_out equals lungmask_b200.laplacian.log_host bit for bit.  d_out, d_work0 and d_work1 must not
 * overlap each other or d_vol.  A NaN or +-inf in the volume returns LM_ERR_NONFINITE (d_out is then not an image). */
LM_API int lm_laplacian_of_gaussian_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2,
                                        const double* spacing_xyz, double sigma_mm, double* d_work0, double* d_work1,
                                        double* d_out, void* stream);

/* Voxel-based first-order feature maps (no counterpart in the reference; DESIGN §4.15): PyRadiomics' voxel-based
 * firstorder extraction of one row, for LMInferer.first_order_maps.  Device memory of the engine's device and the
 * caller's cudaStream_t with the event-wait rule of lm_apply_dev; every argument is checked before any kernel runs and
 * the call returns after the engine's stream has synchronised.  d_vol (n0,n1,n2) of any LM_DTYPE_* code and d_mask
 * (n0,n1,n2) uint8, fewer than 2^32 voxels, never written.  row 1..255 (mask == row) or 256 (mask > 0); the ROI is the
 * row's voxels with a non-NaN value.  radius 1..3: the window of voxel c is the (2 radius + 1)^3 cube about c clipped at
 * the array border; its candidates are the window's ROI voxels (masked 1) or its non-NaN voxels (masked 0).
 * bin_width >= 1, low and n_levels (1..255) the fixed-bin-width discretisation of the host's region; mode
 * LM_FOM_FLOAT, or LM_FOM_EXACT (integer dtypes; every candidate within [base, base + 2^20), |base| <= 2^53);
 * shift: voxelArrayShift, |shift| < 2^58 and, exact, |base + shift| < 2^58.  voxel_volume: the TotalEnergy factor
 * (NaN for none).  feature_bits: a non-empty subset of the 18 bits LM_FOM_* (bit k = first_order.FIRST_ORDER_FEATURES[k]).
 * d_entropy_table: device float64, table_len = K (K + 1) / 2 with K = (2 radius + 1)^3 (see first_order_maps.
 * entropy_table).  d_out: popcount(feature_bits) float64 (n0,n1,n2) planes in bit order, not overlapping the inputs:
 * ROI voxels get their window's features in the sequence of DESIGN §4.15, every other voxel init_value.  A +-inf
 * candidate returns LM_ERR_NONFINITE.  Work area: one flag; each thread holds its window in local memory. */
#define LM_FOM_FLOAT 1
#define LM_FOM_EXACT 2
LM_API int lm_first_order_maps_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                                   int row, int radius, int masked, int bin_width, int64_t low, int n_levels, int mode,
                                   int64_t base, int64_t shift, double voxel_volume, double init_value,
                                   uint32_t feature_bits, const double* d_entropy_table, int64_t table_len, double* d_out,
                                   void* stream);

/* Voxel-based GLCM feature maps (no counterpart in the reference; DESIGN §4.16): PyRadiomics' voxel-based glcm extraction
 * of one row, for LMInferer.glcm_maps.  Device memory of the engine's device and the caller's cudaStream_t with the
 * event-wait rule of lm_apply_dev; every argument is checked before any kernel runs and the call returns after the
 * engine's stream has synchronised.  d_levels (n0,n1,n2) uint8, the level map of lm_texture_levels_dev over the
 * discretisation region (0 outside it), and d_mask (n0,n1,n2) uint8, fewer than 2^32 voxels, never written.  A voxel is
 * a candidate when its level is not 0, and a centre when it is a candidate with mask == row (row 1..255) or mask > 0
 * (row 256).  radius 1..3: the window of a centre is the (2 radius + 1)^3 cube about it clipped at the array border.
 * n_levels 1..255 (Ng of Idmn and Idn); a level above it returns an error and no map.  feature_bits: a non-empty subset
 * of the 22 bits, bit k = texture.GLCM_FEATURES[k].  d_entropy_table: device float64, table_len = M (M + 1) / 2 with
 * M = 2 (2 radius + 1)^2 (2 radius) (see first_order_maps.entropy_table).  d_out: popcount(feature_bits) float64
 * (n0,n1,n2) planes in bit order, not overlapping the inputs: centres get their window's features in the sequence of
 * DESIGN §4.16 (NaN without a pair in any direction), every other voxel init_value.  Work area: one flag; each thread
 * holds its window, pair keys and count tables in local memory. */
LM_API int lm_glcm_maps_dev(lm_engine* e, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2, int row,
                            int radius, int n_levels, double init_value, uint32_t feature_bits,
                            const double* d_entropy_table, int64_t table_len, double* d_out, void* stream);

/* Voxel-based GLSZM, GLRLM, GLDM and NGTDM feature maps (no counterpart in the reference; DESIGN §4.17): PyRadiomics'
 * voxel-based extraction of one texture class of one row, for LMInferer.texture_maps.  Device memory, stream rule,
 * checks, synchronisation, d_levels, d_mask, row, radius and n_levels as for lm_glcm_maps_dev.  A neighbour, run step or
 * zone link counts only when both voxels are candidates of the window.  cls: LM_TEXMAP_GLSZM (zones: 26-connected
 * components of equal level), LM_TEXMAP_GLRLM (runs along the 13 directions, features averaged over them), LM_TEXMAP_GLDM
 * (dependence: neighbours within alpha levels, alpha >= 0; ignored by the other classes) or LM_TEXMAP_NGTDM.
 * feature_bits: a non-empty subset of the class's 16, 16, 14 or 5 bits, bit k = the k-th name of texture.GLSZM_FEATURES,
 * GLRLM_FEATURES, GLDM_FEATURES or NGTDM_FEATURES.  d_entropy_table: device float64, table_len = K (K + 1) / 2 with
 * K = (2 radius + 1)^3 (first_order_maps.entropy_table).  d_out: popcount(feature_bits) float64 (n0,n1,n2) planes in bit
 * order, not overlapping the inputs: centres get their window's features in the sequence of DESIGN §4.17 (NGTDM NaN when
 * no candidate has a neighbour), every other voxel init_value.  Work area: one flag; each thread holds its window, item
 * keys and union-find or per-level tables in local memory. */
#define LM_TEXMAP_GLSZM 1
#define LM_TEXMAP_GLRLM 2
#define LM_TEXMAP_GLDM 3
#define LM_TEXMAP_NGTDM 4
LM_API int lm_texture_maps_dev(lm_engine* e, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2, int row,
                               int radius, int n_levels, int cls, int alpha, double init_value, uint32_t feature_bits,
                               const double* d_entropy_table, int64_t table_len, double* d_out, void* stream);

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
/* The power-of-two scale the split planes of activation `act_id` are stored at in weight slot `slot` (1 until a value
 * of the tensor's scale group left fp16's range; 1 for the fp32 "L" tensors).  lm_load_weights resets it to 1. */
LM_API int lm_debug_activation_scale(lm_engine* e, int slot, int act_id, float* scale);

/* Forward-only benchmark hook: runs the forward pass on `S` device-resident resized slices and
 * reports the device time of the convolution kernels alone (ms) for the roofline. */
LM_API int lm_forward_dev(lm_engine* e, int slot, const int16_t* d_resized, int S, uint8_t* d_labels, float* conv_ms);

#ifdef __cplusplus
}
#endif
#endif /* LUNGMASK_B200_H */
