"""ctypes binding of liblungmask_b200.so (include/lungmask_b200.h).  No torch types cross this boundary."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblungmask_b200.so")

NET_RES = 256
FLAG_NO_POSTPROCESS = 1
DTYPE_I16, DTYPE_F32, DTYPE_F64 = 0, 1, 2   # LM_DTYPE_* of lm_apply_volume_probs
DTYPE_U8, DTYPE_I8, DTYPE_I32, DTYPE_I64, DTYPE_F16, DTYPE_BF16 = 3, 4, 5, 6, 7, 8   # lm_apply_dev only (U8 also bool)
WAVELET_CODES = {"coif1": 0, "haar": 1}   # LM_WAVELET_* of lm_wavelet_dev
ERR_NONFINITE = -41                       # LM_ERR_NONFINITE
FILTER_CODES = {"square": 0, "squareroot": 1, "logarithm": 2, "exponential": 3}   # LM_FILTER_* of lm_image_filter_dev
ERR_TABLE_RANGE = -42                     # LM_ERR_TABLE_RANGE
MESH_RAS = 1                              # LM_MESH_RAS of lm_mesh_emit_dev
FOM_FLOAT, FOM_EXACT = 1, 2               # LM_FOM_* modes of lm_first_order_maps_dev
RESAMPLE_CODES = {"bspline": 0, "nearest": 1}   # LM_RESAMPLE_* of lm_resample_dev

_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    """Loads the CUDA library; fails loudly when it has not been built (there is no CPU fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            "%s is missing: build it with `python -m lungmask_b200.build` (needs nvcc, sm_90a). "
            "lungmask_b200 has no CPU or eager-PyTorch fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32, u8p, i16p, i32p, f32p = C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    sig = {
        "lm_create": ([i32, i32, C.POINTER(vp)], i32),
        "lm_destroy": ([vp], None),
        "lm_last_error": ([], C.c_char_p),
        "lm_device": ([vp], i32),
        "lm_batch_capacity": ([vp], i32),
        "lm_weight_blob_floats": ([i32], C.c_size_t),
        "lm_load_weights": ([vp, i32, f32p, C.c_size_t, i32], i32),
        "lm_apply_volume": ([vp, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_apply_volume_dev": ([vp, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_apply_fused": ([vp, i32, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_apply_fused_dev": ([vp, i32, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_apply_volume_float": ([vp, i32, i32, vp, i32, i32, i32, i32, i32, u8p], i32),
        "lm_preprocess_float": ([vp, vp, i32, i32, i32, i32, f32p, i32p], i32),
        "lm_apply_volume_oriented": ([vp, i32, i32, i16p, i32, i32, i32, vp, vp, i32, u8p], i32),
        "lm_apply_volume_probs": ([vp, i32, vp, i32, i32, i32, i32, vp, vp, i32, u8p, f32p], i32),
        "lm_apply_dev": ([vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, i32, u8p, f32p, vp], i32),
        "lm_label_stats_dev": ([vp, vp, i32, u8p, i32, i32, i32, vp, i32, vp, i32, vp, vp, vp, vp, vp, vp], i32),
        "lm_laa_max_pairs": ([C.c_size_t], C.c_size_t),
        "lm_laa_clusters_dev": ([vp, vp, i32, u8p, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, C.c_size_t, vp], i32),
        "lm_plane_label_counts_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp], i32),
        "lm_surface_distance_dev": ([vp, u8p, i32, i32, i32, vp, vp, vp], i32),
        "lm_region_map_dev": ([vp, u8p, vp, i32, i32, i32, i32, vp, i32, vp, C.c_size_t, vp, vp], i32),
        "lm_texture_levels_dev": ([vp, vp, i32, u8p, i32, i32, i32, i32, C.c_int64, i32, i32, u8p, vp], i32),
        "lm_glcm_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp], i32),
        "lm_zone_sizes_dev": ([vp, u8p, i32, i32, i32, vp, vp, vp, C.c_size_t, vp], i32),
        "lm_glrlm_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp], i32),
        "lm_neighbour_counts_dev": ([vp, u8p, i32, i32, i32, i32, i32, vp, vp, vp, vp], i32),
        "lm_glcm_offsets_dev": ([vp, u8p, i32, i32, i32, i32, vp, i32, vp, vp], i32),
        "lm_neighbour_offsets_dev": ([vp, u8p, i32, i32, i32, i32, i32, vp, i32, vp, vp, vp, vp], i32),
        "lm_zone_sizes_plane_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp, vp, C.c_size_t, vp], i32),
        "lm_shape_sums_dev": ([vp, u8p, i32, i32, i32, vp, vp, vp, vp], i32),
        "lm_max_diameters_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp, vp], i32),
        "lm_mesh_counts_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp, vp, vp, vp], i32),
        "lm_mesh_emit_dev": ([vp, u8p, i32, i32, i32, i32, vp, vp, vp, i32, C.c_int64, C.c_int64, vp, vp, vp, vp], i32),
        "lm_first_order_maps_dev": ([vp, vp, i32, u8p, i32, i32, i32, i32, i32, i32, i32, C.c_int64, i32, i32, C.c_int64,
                                     C.c_int64, C.c_double, C.c_double, C.c_uint32, vp, C.c_int64, vp, vp], i32),
        "lm_glcm_maps_dev": ([vp, u8p, u8p, i32, i32, i32, i32, i32, i32, C.c_double, C.c_uint32, vp, C.c_int64, vp, vp],
                             i32),
        "lm_texture_maps_dev": ([vp, u8p, u8p, i32, i32, i32, i32, i32, i32, i32, i32, C.c_double, C.c_uint32, vp,
                                 C.c_int64, vp, vp], i32),
        "lm_first_order_sums_dev": ([vp, vp, i32, u8p, i32, i32, i32, i32] + [vp] * 12, i32),
        "lm_first_order_splits_dev": ([vp, vp, i32, u8p, i32, i32, i32] + [vp] * 11, i32),
        "lm_wavelet_dev": ([vp, vp, i32, i32, i32, i32, i32, i32, vp, vp], i32),
        "lm_image_range_dev": ([vp, vp, i32, i32, i32, i32, vp, vp], i32),
        "lm_image_filter_dev": ([vp, vp, i32, i32, i32, i32, i32, vp, vp, C.c_int64, C.c_int64, vp, vp], i32),
        "lm_gradient_dev": ([vp, vp, i32, i32, i32, i32, vp, vp, vp], i32),
        "lm_bspline_coefficients_dev": ([vp, vp, i32, i32, i32, i32, vp, vp], i32),
        "lm_resample_dev": ([vp, vp, i32, vp, u8p, i32, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp, u8p, vp], i32),
        "lm_laplacian_of_gaussian_dev": ([vp, vp, i32, i32, i32, i32, vp, C.c_double, vp, vp, vp, vp], i32),
        "lm_shard_init": ([vp, i32, i32, i32], i32),
        "lm_shard_handle_bytes": ([], C.c_size_t),
        "lm_shard_export": ([vp, vp], i32),
        "lm_shard_connect": ([vp, vp], i32),
        "lm_shard_labels": ([vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_size_t)], i32),
        "lm_apply_volume_sharded": ([vp, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_apply_volume_sharded_dev": ([vp, i32, i16p, i32, i32, i32, i32, u8p], i32),
        "lm_fuse": ([vp, u8p, u8p, i32, i32, i32, u8p, C.POINTER(i32)], i32),
        "lm_preprocess": ([vp, i16p, i32, i32, i32, i32, i32, i32, i16p, i32p], i32),
        "lm_simple_bodymask": ([vp, i16p, i32, i32, u8p], i32),
        "lm_forward": ([vp, i32, i16p, i32, u8p, f32p], i32),
        "lm_forward_dev": ([vp, i32, i16p, i32, u8p, C.POINTER(C.c_float)], i32),
        "lm_postprocess": ([vp, u8p, i32, i32, i32, i32p, i32, i32, u8p], i32),
        "lm_reshape_masks": ([vp, u8p, i32, i32, i32p, i32, i32, i32, u8p], i32),
        "lm_keep_largest_component": ([vp, u8p, i32, i32, i32, u8p], i32),
        "lm_last_timings": ([vp, C.POINTER(C.c_float), C.POINTER(C.c_int64)], i32),
        "lm_set_option": ([vp, C.c_char_p, i32], i32),
        "lm_debug_activation_info": ([i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)], i32),
        "lm_debug_read_activation": ([vp, i32, i32, f32p], i32),
        "lm_debug_activation_scale": ([vp, i32, i32, C.POINTER(C.c_float)], i32),
        "lm_last_conv_timing": ([vp, C.POINTER(C.c_float), C.POINTER(C.c_int64)], i32),
    }
    for name, (argtypes, restype) in sig.items():
        fn = getattr(L, name)  # AttributeError here = header / library mismatch
        fn.argtypes, fn.restype = argtypes, restype
    _lib = L
    return L


EXPORTS = ["lm_create", "lm_destroy", "lm_last_error", "lm_device", "lm_batch_capacity", "lm_weight_blob_floats",
           "lm_load_weights", "lm_apply_volume", "lm_apply_volume_dev", "lm_apply_fused", "lm_apply_fused_dev", "lm_apply_volume_oriented", "lm_apply_volume_probs", "lm_apply_dev", "lm_label_stats_dev", "lm_laa_max_pairs", "lm_laa_clusters_dev", "lm_plane_label_counts_dev", "lm_surface_distance_dev", "lm_region_map_dev", "lm_texture_levels_dev", "lm_glcm_dev", "lm_zone_sizes_dev", "lm_glrlm_dev", "lm_neighbour_counts_dev", "lm_glcm_offsets_dev", "lm_neighbour_offsets_dev", "lm_zone_sizes_plane_dev", "lm_shape_sums_dev", "lm_max_diameters_dev", "lm_mesh_counts_dev", "lm_mesh_emit_dev", "lm_first_order_sums_dev", "lm_first_order_splits_dev", "lm_first_order_maps_dev", "lm_glcm_maps_dev", "lm_texture_maps_dev", "lm_wavelet_dev", "lm_image_range_dev", "lm_image_filter_dev", "lm_gradient_dev", "lm_bspline_coefficients_dev", "lm_resample_dev", "lm_laplacian_of_gaussian_dev", "lm_apply_volume_float", "lm_preprocess_float", "lm_fuse", "lm_preprocess",
           "lm_shard_init", "lm_shard_handle_bytes", "lm_shard_export", "lm_shard_connect", "lm_shard_labels",
           "lm_apply_volume_sharded", "lm_apply_volume_sharded_dev",
           "lm_simple_bodymask", "lm_forward", "lm_forward_dev", "lm_postprocess", "lm_reshape_masks",
           "lm_keep_largest_component",
           "lm_last_timings", "lm_set_option", "lm_last_conv_timing",
           "lm_debug_activation_info", "lm_debug_read_activation", "lm_debug_activation_scale"]


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def _check(rc):
    if rc != 0:
        raise NativeError("lungmask_b200 native call failed (%d): %s" % (rc, lib().lm_last_error().decode()))


def _filter_check(rc, what):
    """_check for the filter calls, with a non-finite volume as ValueError."""
    if rc == ERR_NONFINITE:
        raise ValueError("%s: %s" % (what, lib().lm_last_error().decode().split(": ", 1)[1]))
    _check(rc)


def _as(a, dtype, ndim=None):
    """C-contiguous array of `dtype` for the C ABI.  Only value-preserving conversions happen here: a float volume is
    never truncated and an int32 / uint16 volume never wraps silently (integers of another width are range-checked);
    LMInferer / utils do the reference-compatible dtype handling before they get here."""
    a = np.asarray(a)
    dtype = np.dtype(dtype)
    if a.dtype != dtype:
        if a.dtype == bool or np.can_cast(a.dtype, dtype, casting="safe"):
            pass
        elif np.issubdtype(a.dtype, np.integer) and np.issubdtype(dtype, np.integer):
            info = np.iinfo(dtype)
            if a.size and (a.min() < info.min or a.max() > info.max):
                raise TypeError("values of the %s array do not fit %s" % (a.dtype, dtype))
        else:
            raise TypeError("refusing to convert %s to %s (lossy); convert explicitly" % (a.dtype, dtype))
    a = np.ascontiguousarray(a, dtype=dtype)
    if ndim is not None and a.ndim != ndim:
        raise ValueError("expected %d-d array, got shape %s" % (ndim, a.shape))
    return a


class Engine:
    """One engine = one CUDA device (see lm_create)."""

    def __init__(self, device=0, batch_capacity=20):
        self._h = C.c_void_p()
        _check(lib().lm_create(int(device), int(batch_capacity), C.byref(self._h)))
        self.device, self.batch_capacity = int(device), int(batch_capacity)
        self.n_classes = {}

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().lm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights
    def load_weights(self, slot, blob, n_classes):
        blob = _as(blob, np.float32, 1)
        _check(lib().lm_load_weights(self._h, slot, _ptr(blob), blob.size, int(n_classes)))
        self.n_classes[slot] = int(n_classes)

    # ---- whole path
    def apply_volume(self, slot, vol, postprocess=True, out=None):
        vol = _as(vol, np.int16, 3)
        if out is None:
            out = np.empty(vol.shape, np.uint8)
        assert out.dtype == np.uint8 and out.shape == vol.shape and out.flags.c_contiguous
        S, H, W = vol.shape
        _check(lib().lm_apply_volume(self._h, slot, _ptr(vol), S, H, W, 0 if postprocess else FLAG_NO_POSTPROCESS, _ptr(out)))
        return out

    def apply_volume_dev(self, slot, d_vol_ptr, shape, d_out_ptr, postprocess=True):
        S, H, W = shape
        _check(lib().lm_apply_volume_dev(self._h, slot, C.c_void_p(d_vol_ptr), S, H, W,
                                         0 if postprocess else FLAG_NO_POSTPROCESS, C.c_void_p(d_out_ptr)))

    def apply_fused(self, slot_base, slot_fill, vol, postprocess=True):
        """`postprocess` = LMInferer.volume_postprocessing: it reaches the two inner inferences only (mask.py:191-194);
        the fusion post-processing (mask.py:232) always runs."""
        vol = _as(vol, np.int16, 3)
        out = np.empty(vol.shape, np.uint8)
        S, H, W = vol.shape
        _check(lib().lm_apply_fused(self._h, slot_base, slot_fill, _ptr(vol), S, H, W,
                                    0 if postprocess else FLAG_NO_POSTPROCESS, _ptr(out)))
        return out

    def apply_fused_dev(self, slot_base, slot_fill, d_vol_ptr, shape, d_out_ptr, postprocess=True):
        S, H, W = shape
        _check(lib().lm_apply_fused_dev(self._h, slot_base, slot_fill, C.c_void_p(d_vol_ptr), S, H, W,
                                        0 if postprocess else FLAG_NO_POSTPROCESS, C.c_void_p(d_out_ptr)))

    def apply_volume_float(self, slot, vol, slot_fill=-1, postprocess=True):
        """float32 / float64 HU volume (the dtype is kept through pre-processing and normalisation, as the reference does)."""
        vol = np.asarray(vol)
        if vol.dtype not in (np.float32, np.float64):
            raise TypeError("apply_volume_float expects float32 or float64, got %s" % vol.dtype)
        vol = _as(vol, vol.dtype, 3)
        out = np.empty(vol.shape, np.uint8)
        S, H, W = vol.shape
        _check(lib().lm_apply_volume_float(self._h, slot, int(slot_fill), _ptr(vol), 1 if vol.dtype == np.float64 else 0, S, H, W,
                                           0 if postprocess else FLAG_NO_POSTPROCESS, _ptr(out)))
        return out

    def preprocess_float(self, vol):
        vol = np.asarray(vol)
        if vol.dtype not in (np.float32, np.float64):
            raise TypeError("preprocess_float expects float32 or float64, got %s" % vol.dtype)
        vol = _as(vol, vol.dtype, 3)
        S, H, W = vol.shape
        norm = np.empty((S, NET_RES, NET_RES), np.float32)
        boxes = np.empty((S, 4), np.int32)
        _check(lib().lm_preprocess_float(self._h, _ptr(vol), 1 if vol.dtype == np.float64 else 0, S, H, W, _ptr(norm), _ptr(boxes)))
        return norm, boxes

    def apply_volume_oriented(self, slot, vol, perm, flip, slot_fill=-1, postprocess=True):
        """`vol` in its native orientation; (perm, flip) = lungmask_b200.orient.array_transform_to_lps(code)."""
        vol = _as(vol, np.int16, 3)
        out = np.empty(vol.shape, np.uint8)
        pa = (C.c_int * 3)(*[int(x) for x in perm])
        fa = (C.c_int * 3)(*[1 if x else 0 for x in flip])
        n0, n1, n2 = vol.shape
        _check(lib().lm_apply_volume_oriented(self._h, slot, int(slot_fill), _ptr(vol), n0, n1, n2, pa, fa,
                                              0 if postprocess else FLAG_NO_POSTPROCESS, _ptr(out)))
        return out

    def apply_volume_probs(self, slot, vol, perm=None, flip=None, postprocess=True):
        """-> (mask, probs) of one model from one forward pass (lm_apply_volume_probs).  `vol`: int16 (other integer
        widths must fit int16), float32 or float64, in its native orientation; (perm, flip) =
        lungmask_b200.orient.array_transform_to_lps(code), or both None for an LPS array.  `mask` (uint8, vol.shape) is
        what apply_volume / apply_volume_float / apply_volume_oriented return with the same `postprocess`.  `probs`
        (float32, (K,) + vol.shape) are the network's class probabilities BEFORE post-processing, resampled to the
        input like the mask (order 0, p_0 = 1 outside the crop box)."""
        vol = np.asarray(vol)
        if vol.dtype == np.float32 or vol.dtype == np.float64:
            dtype = DTYPE_F32 if vol.dtype == np.float32 else DTYPE_F64
            vol = _as(vol, vol.dtype, 3)
        else:
            dtype = DTYPE_I16
            vol = _as(vol, np.int16, 3)
        if (perm is None) != (flip is None):
            raise ValueError("apply_volume_probs: give both perm and flip, or neither")
        if slot not in self.n_classes:
            raise NativeError("apply_volume_probs: weight slot %d not loaded" % slot)
        out = np.empty(vol.shape, np.uint8)
        probs = np.empty((self.n_classes[slot],) + vol.shape, np.float32)
        pa = fa = None
        if perm is not None:
            pa = (C.c_int * 3)(*[int(x) for x in perm])
            fa = (C.c_int * 3)(*[1 if x else 0 for x in flip])
        n0, n1, n2 = vol.shape
        _check(lib().lm_apply_volume_probs(self._h, slot, _ptr(vol), dtype, n0, n1, n2, pa, fa,
                                           0 if postprocess else FLAG_NO_POSTPROCESS, _ptr(out), _ptr(probs)))
        return out, probs

    def apply_dev(self, slot, d_vol_ptr, dtype_code, shape, d_out_ptr, perm=None, flip=None, slot_fill=-1, d_probs_ptr=None,
                  postprocess=True, stream=0):
        """lm_apply_dev: the whole path on device memory of this engine's device.  `d_vol_ptr`: a C-contiguous `shape`
        volume of element type `dtype_code` (DTYPE_*) in its native orientation; (perm, flip) as for apply_volume_probs.
        Writes the uint8 mask to `d_out_ptr` and, if given, the (K,) + shape float32 probabilities to `d_probs_ptr` (not
        with slot_fill >= 0).  `stream`: the caller's cudaStream_t as an int (0 = the legacy default stream); the engine
        waits for the work queued on it before it reads the volume, and the results are complete when this returns."""
        if (perm is None) != (flip is None):
            raise ValueError("apply_dev: give both perm and flip, or neither")
        pa = fa = None
        if perm is not None:
            pa = (C.c_int * 3)(*[int(x) for x in perm])
            fa = (C.c_int * 3)(*[1 if x else 0 for x in flip])
        n0, n1, n2 = (int(x) for x in shape)
        _check(lib().lm_apply_dev(self._h, int(slot), int(slot_fill), C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2, pa, fa,
                                  0 if postprocess else FLAG_NO_POSTPROCESS, C.c_void_p(d_out_ptr),
                                  C.c_void_p(d_probs_ptr) if d_probs_ptr else None, C.c_void_p(int(stream)) if stream else None))

    # ---- per-label statistics (lm_label_stats_dev)
    def label_stats_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, percentiles=(15.0,), thresholds=(-950,), stream=0):
        """lm_label_stats_dev on device memory of this engine's device (`stream` as for apply_dev) -> dict of numpy arrays
        over 257 rows (row l = label l, row 256 = the union mask > 0): "voxels", "nan_voxels" (int64), "moments" (257, 4)
        mean / std / min / max, "percentile" (257, n_q), "below_count" (257, n_t) int64."""
        n0, n1, n2 = (int(x) for x in shape)
        q = np.ascontiguousarray(percentiles, dtype=np.float64).reshape(-1)
        t = np.ascontiguousarray(thresholds, dtype=np.int32).reshape(-1)
        res = {"voxels": np.zeros(257, np.int64), "nan_voxels": np.zeros(257, np.int64),
               "moments": np.zeros((257, 4), np.float64), "percentile": np.zeros((257, max(q.size, 1)), np.float64),
               "below_count": np.zeros((257, max(t.size, 1)), np.int64)}
        _check(lib().lm_label_stats_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr), n0, n1, n2,
                                        _ptr(q), q.size, _ptr(t), t.size, _ptr(res["voxels"]), _ptr(res["nan_voxels"]),
                                        _ptr(res["moments"]), _ptr(res["percentile"]), _ptr(res["below_count"]),
                                        C.c_void_p(int(stream)) if stream else None))
        res["percentile"] = res["percentile"][:, :q.size]
        res["below_count"] = res["below_count"][:, :t.size]
        return res

    # ---- LAA cluster size distributions (lm_laa_clusters_dev)
    def laa_clusters_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, threshold=-950, connectivity=6, stream=0):
        """lm_laa_clusters_dev on device memory of this engine's device (`stream` as for apply_dev) -> dict over 257 rows
        (row l = label l, row 256 = all LAA voxels): "laa_voxels", "n_clusters", "n_pairs" (int64 [257]) and "sizes",
        "counts" (int64, the rows' (size, count) pairs concatenated; row r's are [offsets[r], offsets[r + 1])), "offsets"."""
        n0, n1, n2 = (int(x) for x in shape)
        cap = int(lib().lm_laa_max_pairs(max(n0, 0) * max(n1, 0) * max(n2, 0)))
        res = {k: np.zeros(257, np.int64) for k in ("laa_voxels", "n_clusters", "n_pairs")}
        sizes, counts = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
        _check(lib().lm_laa_clusters_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr), n0, n1, n2,
                                         int(threshold), int(connectivity), _ptr(res["laa_voxels"]), _ptr(res["n_clusters"]),
                                         _ptr(res["n_pairs"]), _ptr(sizes), _ptr(counts), cap,
                                         C.c_void_p(int(stream)) if stream else None))
        res["offsets"] = np.concatenate([[0], np.cumsum(res["n_pairs"])])
        total = int(res["offsets"][-1])
        res["sizes"], res["counts"] = sizes[:total].copy(), counts[:total].copy()
        return res

    # ---- regional statistics support (lm_plane_label_counts_dev, lm_surface_distance_dev, lm_region_map_dev)
    def plane_label_counts_dev(self, d_mask_ptr, shape, axis, stream=0):
        """Voxels per label in every plane along array `axis` of a (n0,n1,n2) uint8 device mask (`stream` as for apply_dev)
        -> int64 (n_axis, 257): [p, l] = voxels with mask == l in plane p, [p, 256] = mask > 0."""
        n0, n1, n2 = (int(x) for x in shape)
        n_axis = (n0, n1, n2)[axis] if axis in (0, 1, 2) else 0
        counts = np.zeros((max(n_axis, 1), 257), np.int64)
        _check(lib().lm_plane_label_counts_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, int(axis), _ptr(counts),
                                               C.c_void_p(int(stream)) if stream else None))
        return counts[:n_axis]

    def surface_distance_dev(self, d_mask_ptr, shape, spacing, d_out_ptr, stream=0):
        """Writes the float32 distance (mm) of every mask > 0 voxel to the nearest mask == 0 voxel to `d_out_ptr`;
        `spacing` per array axis (s0, s1, s2)."""
        n0, n1, n2 = (int(x) for x in shape)
        sp = np.ascontiguousarray(spacing, dtype=np.float64).reshape(-1)
        if sp.size != 3:
            raise ValueError("surface_distance_dev: spacing needs 3 values, got %d" % sp.size)
        _check(lib().lm_surface_distance_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, _ptr(sp), C.c_void_p(d_out_ptr),
                                             C.c_void_p(int(stream)) if stream else None))

    def region_map_dev(self, d_mask_ptr, shape, lut, d_map_ptr, axis=None, d_dist_ptr=None, bounds=(), stream=0):
        """Writes d_map[v] = lut[bucket(v), mask[v]]: bucket = the plane index along `axis` (d_dist_ptr None) or the
        number of the float32 `bounds` <= d_dist[v].  `lut`: uint8 (buckets, 256) with lut[:, 0] == 0."""
        n0, n1, n2 = (int(x) for x in shape)
        lut = np.ascontiguousarray(lut, dtype=np.uint8)
        b = np.ascontiguousarray(bounds, dtype=np.float32).reshape(-1)
        _check(lib().lm_region_map_dev(self._h, C.c_void_p(d_mask_ptr), C.c_void_p(d_dist_ptr) if d_dist_ptr else None,
                                       n0, n1, n2, -1 if axis is None else int(axis), _ptr(b) if b.size else None, int(b.size),
                                       _ptr(lut), lut.size, C.c_void_p(d_map_ptr), C.c_void_p(int(stream)) if stream else None))

    # ---- texture matrices (lm_texture_levels_dev, lm_glcm_dev, lm_zone_sizes_dev, lm_glrlm_dev, lm_neighbour_counts_dev)
    def texture_levels_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, row, low, bin_width, n_levels, d_levels_ptr, stream=0):
        """Writes the uint8 level map of `row` (1..255, or 256 for mask > 0) to `d_levels_ptr` (16-byte aligned):
        floor((floor(x) - low) / bin_width) + 1 on the row's non-NaN voxels, 0 elsewhere (`stream` as for apply_dev)."""
        n0, n1, n2 = (int(x) for x in shape)
        _check(lib().lm_texture_levels_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr), n0, n1, n2,
                                           int(row), int(low), int(bin_width), int(n_levels), C.c_void_p(d_levels_ptr),
                                           C.c_void_p(int(stream)) if stream else None))

    def glcm_dev(self, d_levels_ptr, shape, n_levels, stream=0):
        """-> int64 (13, n_levels (n_levels + 1) / 2): the unordered pair counts U_d(i <= j) of a uint8 level map, in the
        direction order of lm_glcm_dev and the order of np.triu_indices(n_levels)."""
        n0, n1, n2 = (int(x) for x in shape)
        ng = int(n_levels)
        counts = np.zeros((13, max(ng * (ng + 1) // 2, 1)), np.int64)
        _check(lib().lm_glcm_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, ng, _ptr(counts),
                                 C.c_void_p(int(stream)) if stream else None))
        return counts

    def zone_sizes_dev(self, d_levels_ptr, shape, stream=0):
        """-> dict: "n_pairs" (int64 [256], row = level), "sizes", "counts" (the rows' (size, count) pairs concatenated;
        row r's are [offsets[r], offsets[r + 1])), "offsets": the 26-connected zones of equal level of a uint8 level map."""
        n0, n1, n2 = (int(x) for x in shape)
        cap = int(lib().lm_laa_max_pairs(max(n0, 0) * max(n1, 0) * max(n2, 0)))
        n_pairs = np.zeros(256, np.int64)
        sizes, counts = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
        _check(lib().lm_zone_sizes_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, _ptr(n_pairs), _ptr(sizes), _ptr(counts),
                                       cap, C.c_void_p(int(stream)) if stream else None))
        offsets = np.concatenate([[0], np.cumsum(n_pairs)])
        total = int(offsets[-1])
        return {"n_pairs": n_pairs, "sizes": sizes[:total].copy(), "counts": counts[:total].copy(), "offsets": offsets}

    def glrlm_dev(self, d_levels_ptr, shape, n_levels, stream=0):
        """-> int64 (13, n_levels, max(shape)): the runs of level i + 1 and length k + 1 of a uint8 level map along each
        direction d of lm_glcm_dev."""
        n0, n1, n2 = (int(x) for x in shape)
        ng = int(n_levels)
        counts = np.zeros((13, max(ng, 1), max(n0, n1, n2, 1)), np.int64)
        _check(lib().lm_glrlm_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, ng, _ptr(counts),
                                  C.c_void_p(int(stream)) if stream else None))
        return counts

    def neighbour_counts_dev(self, d_levels_ptr, shape, n_levels, alpha=0, stream=0):
        """-> (G, N, A), each int64 (n_levels, 27), of a uint8 level map: G(i, c) the voxels of level i + 1 with c
        neighbours in the ROI within `alpha` levels, N(i, W) those with W neighbours in the ROI, A(i, W) the sum of
        |W (i + 1) - S| over them (S the sum of the neighbours' levels)."""
        n0, n1, n2 = (int(x) for x in shape)
        ng = int(n_levels)
        G, N, A = (np.zeros((max(ng, 1), 27), np.int64) for _ in range(3))
        _check(lib().lm_neighbour_counts_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, ng, int(alpha), _ptr(G), _ptr(N),
                                             _ptr(A), C.c_void_p(int(stream)) if stream else None))
        return G, N, A

    # ---- generalised neighbourhoods (lm_glcm_offsets_dev, lm_neighbour_offsets_dev, lm_zone_sizes_plane_dev)
    def glcm_offsets_dev(self, d_levels_ptr, shape, n_levels, offsets, stream=0):
        """-> int64 (len(offsets), n_levels (n_levels + 1) / 2): the unordered pair counts U_o(i <= j) of a uint8 level
        map for each (dz, dy, dx) of `offsets` (texture.offsets), in their order and the order of np.triu_indices."""
        n0, n1, n2 = (int(x) for x in shape)
        ng = int(n_levels)
        o = np.ascontiguousarray(offsets, dtype=np.int8).reshape(-1, 3)
        counts = np.zeros((max(len(o), 1), max(ng * (ng + 1) // 2, 1)), np.int64)
        _check(lib().lm_glcm_offsets_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, ng, _ptr(o), len(o), _ptr(counts),
                                         C.c_void_p(int(stream)) if stream else None))
        return counts

    def neighbour_offsets_dev(self, d_levels_ptr, shape, n_levels, offsets, alpha=0, stream=0):
        """-> (G, N, A), each int64 (n_levels, 2 len(offsets) + 1): neighbour_counts_dev over the neighbourhood
        v +- o for o in `offsets`."""
        n0, n1, n2 = (int(x) for x in shape)
        ng = int(n_levels)
        o = np.ascontiguousarray(offsets, dtype=np.int8).reshape(-1, 3)
        G, N, A = (np.zeros((max(ng, 1), 2 * len(o) + 1), np.int64) for _ in range(3))
        _check(lib().lm_neighbour_offsets_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, ng, int(alpha), _ptr(o), len(o),
                                              _ptr(G), _ptr(N), _ptr(A), C.c_void_p(int(stream)) if stream else None))
        return G, N, A

    def zone_sizes_plane_dev(self, d_levels_ptr, shape, axis, stream=0):
        """zone_sizes_dev with zones 8-connected within each plane normal to `axis` (0, 1 or 2)."""
        n0, n1, n2 = (int(x) for x in shape)
        cap = int(lib().lm_laa_max_pairs(max(n0, 0) * max(n1, 0) * max(n2, 0)))
        n_pairs = np.zeros(256, np.int64)
        sizes, counts = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
        _check(lib().lm_zone_sizes_plane_dev(self._h, C.c_void_p(d_levels_ptr), n0, n1, n2, int(axis), _ptr(n_pairs),
                                             _ptr(sizes), _ptr(counts), cap, C.c_void_p(int(stream)) if stream else None))
        offsets = np.concatenate([[0], np.cumsum(n_pairs)])
        total = int(offsets[-1])
        return {"n_pairs": n_pairs, "sizes": sizes[:total].copy(), "counts": counts[:total].copy(), "offsets": offsets}

    # ---- mesh shape support (lm_shape_sums_dev, lm_max_diameters_dev)
    def shape_sums_dev(self, d_mask_ptr, shape, stream=0):
        """-> dict over 257 rows (row l = mask == l, row 256 = mask != 0) of a (n0,n1,n2) uint8 device mask padded with
        outside: "cube_counts" int64 (257, 256) marching-cube configurations, "cube_possum" int64 (257, 256, 3) the sums of
        their lowest corners, "moments" int64 (257, 10) (`stream` as for apply_dev)."""
        n0, n1, n2 = (int(x) for x in shape)
        res = {"cube_counts": np.zeros((257, 256), np.int64), "cube_possum": np.zeros((257, 256, 3), np.int64),
               "moments": np.zeros((257, 10), np.int64)}
        _check(lib().lm_shape_sums_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, _ptr(res["cube_counts"]),
                                       _ptr(res["cube_possum"]), _ptr(res["moments"]), C.c_void_p(int(stream)) if stream else None))
        return res

    def max_diameters_dev(self, d_mask_ptr, shape, row, spacing, stream=0):
        """-> float64 [4]: the largest squared distances (mm^2) between mesh vertices of `row` (1..255, or 256 for
        mask != 0) - all pairs, equal axis-0, axis-1, axis-2 coordinate; `spacing` per array axis (s0, s1, s2)."""
        n0, n1, n2 = (int(x) for x in shape)
        sp = np.ascontiguousarray(spacing, dtype=np.float64).reshape(-1)
        if sp.size != 3:
            raise ValueError("max_diameters_dev: spacing needs 3 values, got %d" % sp.size)
        d2 = np.zeros(4, np.float64)
        _check(lib().lm_max_diameters_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, int(row), _ptr(sp), _ptr(d2),
                                          C.c_void_p(int(stream)) if stream else None))
        return d2

    # ---- surface meshes (lm_mesh_counts_dev, lm_mesh_emit_dev)
    def mesh_counts_dev(self, d_mask_ptr, shape, row, tri_offsets, tri_codes, stream=0):
        """-> (V, T): the vertices and triangles of the marching-cubes mesh of `row` (1..255, or 256 for mask != 0) of a
        (n0,n1,n2) uint8 device mask padded with outside, for the table (tri_offsets int32 [257], tri_codes uint8
        [3 tri_offsets[256]] of (corner << 2) | axis codes; `stream` as for apply_dev)."""
        n0, n1, n2 = (int(x) for x in shape)
        off, codes = _as(tri_offsets, np.int32, 1), _as(tri_codes, np.uint8, 1)
        nv, nt = C.c_int64(0), C.c_int64(0)
        _check(lib().lm_mesh_counts_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, int(row), _ptr(off), _ptr(codes),
                                        C.byref(nv), C.byref(nt), C.c_void_p(int(stream)) if stream else None))
        return int(nv.value), int(nt.value)

    def mesh_emit_dev(self, d_mask_ptr, shape, row, tri_offsets, tri_codes, geometry, n_vertices, n_triangles, d_index2_ptr,
                      d_vertices_ptr, d_triangles_ptr, ras=False, stream=0):
        """Writes the mesh of `row` (counts from mesh_counts_dev): int32 (V,3) doubled coordinates, float64 (V,3) positions
        and int32 (T,3) vertex indices to the device pointers.  `geometry`: 15 float64, origin (3), direction (9, row-major)
        and spacing (x, y, z); `ras` negates the first two components."""
        n0, n1, n2 = (int(x) for x in shape)
        off, codes = _as(tri_offsets, np.int32, 1), _as(tri_codes, np.uint8, 1)
        geo = np.ascontiguousarray(geometry, dtype=np.float64).reshape(-1)
        if geo.size != 15:
            raise ValueError("mesh_emit_dev: geometry needs 15 values, got %d" % geo.size)
        _check(lib().lm_mesh_emit_dev(self._h, C.c_void_p(d_mask_ptr), n0, n1, n2, int(row), _ptr(off), _ptr(codes), _ptr(geo),
                                      MESH_RAS if ras else 0, int(n_vertices), int(n_triangles),
                                      C.c_void_p(d_index2_ptr or None), C.c_void_p(d_vertices_ptr or None),
                                      C.c_void_p(d_triangles_ptr or None), C.c_void_p(int(stream)) if stream else None))

    # ---- voxel-based first-order maps (lm_first_order_maps_dev)
    def first_order_maps_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, row, radius, masked, bin_width, low, n_levels,
                             exact, base, shift, voxel_volume, init_value, feature_bits, d_table_ptr, table_len, d_out_ptr,
                             stream=0):
        """Writes the popcount(feature_bits) float64 maps of `row` (1..255, or 256 for mask > 0) to d_out (device memory of
        this engine's device; `stream` as for apply_dev).  A +-inf in a window is a ValueError."""
        n0, n1, n2 = (int(x) for x in shape)
        _filter_check(lib().lm_first_order_maps_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr),
                                                    n0, n1, n2, int(row), int(radius), int(bool(masked)), int(bin_width),
                                                    int(low), int(n_levels), FOM_EXACT if exact else FOM_FLOAT, int(base),
                                                    int(shift), float(voxel_volume), float(init_value), int(feature_bits),
                                                    C.c_void_p(d_table_ptr), int(table_len), C.c_void_p(d_out_ptr),
                                                    C.c_void_p(int(stream)) if stream else None), "first_order_maps")

    # ---- voxel-based GLCM maps (lm_glcm_maps_dev)
    def glcm_maps_dev(self, d_levels_ptr, d_mask_ptr, shape, row, radius, n_levels, init_value, feature_bits, d_table_ptr,
                      table_len, d_out_ptr, stream=0):
        """Writes the popcount(feature_bits) float64 GLCM maps of `row` (1..255, or 256 for mask > 0) of a level map to
        d_out (device memory of this engine's device; `stream` as for apply_dev)."""
        n0, n1, n2 = (int(x) for x in shape)
        _check(lib().lm_glcm_maps_dev(self._h, C.c_void_p(d_levels_ptr), C.c_void_p(d_mask_ptr), n0, n1, n2, int(row),
                                      int(radius), int(n_levels), float(init_value), int(feature_bits),
                                      C.c_void_p(d_table_ptr), int(table_len), C.c_void_p(d_out_ptr),
                                      C.c_void_p(int(stream)) if stream else None))

    # ---- voxel-based GLSZM / GLRLM / GLDM / NGTDM maps (lm_texture_maps_dev)
    def texture_maps_dev(self, d_levels_ptr, d_mask_ptr, shape, row, radius, n_levels, cls, alpha, init_value, feature_bits,
                         d_table_ptr, table_len, d_out_ptr, stream=0):
        """Writes the popcount(feature_bits) float64 maps of texture class `cls` (texture_maps.CLASS_CODES) of `row` (1..255, or 256 for
        mask > 0) of a level map to d_out (device memory of this engine's device; `stream` as for apply_dev)."""
        n0, n1, n2 = (int(x) for x in shape)
        _check(lib().lm_texture_maps_dev(self._h, C.c_void_p(d_levels_ptr), C.c_void_p(d_mask_ptr), n0, n1, n2, int(row),
                                         int(radius), int(n_levels), int(cls), int(alpha), float(init_value),
                                         int(feature_bits), C.c_void_p(d_table_ptr), int(table_len),
                                         C.c_void_p(d_out_ptr), C.c_void_p(int(stream)) if stream else None))

    # ---- first-order sums (lm_first_order_sums_dev, lm_first_order_splits_dev)
    @staticmethod
    def _rows(values, dtype):
        """A per-row input of the first-order calls: 257 values (row 0 unused) as a C-contiguous host array."""
        a = np.ascontiguousarray(values, dtype=dtype).reshape(-1)
        if a.size != 257:
            raise ValueError("first-order row inputs need 257 values (rows 0..256), got %d" % a.size)
        return a

    def first_order_sums_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, bin_width, mode, low, n_levels, base, centre,
                             band_lo, band_hi, stream=0):
        """lm_first_order_sums_dev (pass A) on device memory of this engine's device (`stream` as for apply_dev); every row
        input has 257 entries -> dict: "histogram" int64 (257, 256), "int_sums" uint64 (257, 10) (S1..S4, S_B as (low,
        high) word pairs of exact rows), "band_count" int64 [257], "float_sums" float64 (257, 5) (float rows)."""
        n0, n1, n2 = (int(x) for x in shape)
        ins = [self._rows(mode, np.int32), self._rows(low, np.int64), self._rows(n_levels, np.int32),
               self._rows(base, np.int64), self._rows(centre, np.float64), self._rows(band_lo, np.float64),
               self._rows(band_hi, np.float64)]
        res = {"histogram": np.zeros((257, 256), np.int64), "int_sums": np.zeros((257, 10), np.uint64),
               "band_count": np.zeros(257, np.int64), "float_sums": np.zeros((257, 5), np.float64)}
        _check(lib().lm_first_order_sums_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr), n0, n1,
                                             n2, int(bin_width), *[_ptr(a) for a in ins],
                                             *[_ptr(res[k]) for k in ("histogram", "int_sums", "band_count", "float_sums")],
                                             C.c_void_p(int(stream)) if stream else None))
        return res

    def first_order_splits_dev(self, d_vol_ptr, dtype_code, d_mask_ptr, shape, mode, base, split, split_band, centre,
                               centre_band, band_lo, band_hi, stream=0):
        """lm_first_order_splits_dev (pass B), row inputs as for first_order_sums_dev -> dict: "below" int64 (257, 4)
        (n_lo, L, n_lo_B, L_B of exact rows), "abs_dev" float64 (257, 2) (float rows)."""
        n0, n1, n2 = (int(x) for x in shape)
        ins = [self._rows(mode, np.int32), self._rows(base, np.int64), self._rows(split, np.int64),
               self._rows(split_band, np.int64), self._rows(centre, np.float64), self._rows(centre_band, np.float64),
               self._rows(band_lo, np.float64), self._rows(band_hi, np.float64)]
        res = {"below": np.zeros((257, 4), np.int64), "abs_dev": np.zeros((257, 2), np.float64)}
        _check(lib().lm_first_order_splits_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_mask_ptr), n0,
                                               n1, n2, *[_ptr(a) for a in ins], _ptr(res["below"]), _ptr(res["abs_dev"]),
                                               C.c_void_p(int(stream)) if stream else None))
        return res

    # ---- wavelet decomposition (lm_wavelet_dev)
    def wavelet_dev(self, d_vol_ptr, dtype_code, shape, wavelet, band, d_out_ptr, stream=0):
        """Writes band `band` (0..7 = 4 h_x + 2 h_y + h_z) of the `wavelet` ("coif1" or "haar") decomposition of a
        C-contiguous `shape` device volume of element type `dtype_code` to the float64 `shape` device buffer `d_out_ptr`
        (`stream` as for apply_dev).  ValueError when the volume holds a NaN or +-inf; NativeError for the other failures."""
        n0, n1, n2 = (int(x) for x in shape)
        if wavelet not in WAVELET_CODES:
            raise ValueError("wavelet_dev: unknown wavelet %r (known: %s)" % (wavelet, ", ".join(WAVELET_CODES)))
        rc = lib().lm_wavelet_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2, WAVELET_CODES[wavelet],
                                  int(band), C.c_void_p(d_out_ptr), C.c_void_p(int(stream)) if stream else None)
        if rc == ERR_NONFINITE:
            raise ValueError("wavelet: " + lib().lm_last_error().decode().split(": ", 1)[1])
        _check(rc)

    # ---- image filters (lm_image_range_dev, lm_image_filter_dev, lm_gradient_dev)
    def image_range_dev(self, d_vol_ptr, dtype_code, shape, stream=0):
        """(min, max) of a C-contiguous `shape` device volume of element type `dtype_code`, every voxel as float64
        (`stream` as for apply_dev).  ValueError when the volume holds a NaN or +-inf; NativeError for the other
        failures."""
        n0, n1, n2 = (int(x) for x in shape)
        out = np.zeros(2, np.float64)
        rc = lib().lm_image_range_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2, _ptr(out),
                                      C.c_void_p(int(stream)) if stream else None)
        _filter_check(rc, "image range")
        return float(out[0]), float(out[1])

    def image_filter_dev(self, d_vol_ptr, dtype_code, shape, image_type, param, d_out_ptr, table=None, stream=0):
        """Writes the elementwise image type `image_type` ("square", "squareroot", "logarithm", "exponential") of a
        C-contiguous `shape` device volume to the float64 `shape` device buffer `d_out_ptr`: with the host scalar
        `param`, or, when `table` = (device pointer of a float64 table, its first value, its length) is given, as
        table[x - first value].  ValueError when the volume holds a NaN or +-inf; NativeError for the other failures."""
        n0, n1, n2 = (int(x) for x in shape)
        if image_type not in FILTER_CODES:
            raise ValueError("image_filter_dev: unknown image type %r (known: %s)" % (image_type, ", ".join(FILTER_CODES)))
        params = np.array([param], np.float64)
        d_table, table_min, table_len = table if table is not None else (0, 0, 0)
        rc = lib().lm_image_filter_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2,
                                       FILTER_CODES[image_type], _ptr(params), C.c_void_p(d_table or None),
                                       int(table_min), int(table_len), C.c_void_p(d_out_ptr),
                                       C.c_void_p(int(stream)) if stream else None)
        _filter_check(rc, image_type)

    def gradient_dev(self, d_vol_ptr, dtype_code, shape, spacing_xyz, d_out_ptr, stream=0):
        """Writes the gradient magnitude (ITK's GradientMagnitudeImageFilter, spacing (x, y, z) in mm) of a
        C-contiguous `shape` device volume to the float64 `shape` device buffer `d_out_ptr`.  ValueError when the volume
        holds a NaN or +-inf; NativeError for the other failures."""
        n0, n1, n2 = (int(x) for x in shape)
        sp = np.array([float(s) for s in spacing_xyz], np.float64)
        rc = lib().lm_gradient_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2, _ptr(sp),
                                   C.c_void_p(d_out_ptr), C.c_void_p(int(stream)) if stream else None)
        _filter_check(rc, "gradient")

    # ---- resampling (lm_bspline_coefficients_dev, lm_resample_dev)
    @staticmethod
    def _resample_check(rc, what):
        """ValueError for an argument refused by the call or a NaN or +-inf; NativeError for a CUDA failure."""
        if rc in (-1, ERR_NONFINITE):
            raise ValueError("%s: %s" % (what, lib().lm_last_error().decode()))
        _check(rc)

    def bspline_coefficients_dev(self, d_vol_ptr, dtype_code, shape, d_coeff_ptr, stream=0):
        """Writes the float64 cubic B-spline coefficients (mirror boundaries) of a C-contiguous `shape` device volume of
        element type `dtype_code` to the float64 `shape` device buffer `d_coeff_ptr` (`stream` as for apply_dev).
        ValueError for a refused argument or a NaN or +-inf in the volume; NativeError for the other failures."""
        n0, n1, n2 = (int(x) for x in shape)
        rc = lib().lm_bspline_coefficients_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2,
                                               C.c_void_p(d_coeff_ptr), C.c_void_p(int(stream)) if stream else None)
        self._resample_check(rc, "bspline_coefficients")

    def resample_dev(self, d_vol_ptr, dtype_code, d_coeff_ptr, d_mask_ptr, shape, d_tables, out_shape, interpolator,
                     d_out_ptr, d_out_mask_ptr, stream=0):
        """Samples a C-contiguous `shape` device volume (element type `dtype_code`) and its uint8 mask on the `out_shape`
        grid of the device float64 tables d_tables = (c_z, c_y, c_x) pointers: the image into `d_out_ptr` (the volume's
        dtype) from the coefficients `d_coeff_ptr` ("bspline") or the volume ("nearest"), the mask into the uint8
        `d_out_mask_ptr`.  ValueError for a refused argument or a NaN or +-inf sample; NativeError for the other
        failures."""
        n0, n1, n2 = (int(x) for x in shape)
        m0, m1, m2 = (int(x) for x in out_shape)
        if interpolator not in RESAMPLE_CODES:
            raise ValueError("resample_dev: unknown interpolator %r (known: %s)" % (interpolator, ", ".join(RESAMPLE_CODES)))
        cz, cy, cx = (C.c_void_p(int(p)) for p in d_tables)
        rc = lib().lm_resample_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), C.c_void_p(d_coeff_ptr or None),
                                   C.c_void_p(d_mask_ptr), n0, n1, n2, cz, cy, cx, m0, m1, m2, RESAMPLE_CODES[interpolator],
                                   C.c_void_p(d_out_ptr), C.c_void_p(d_out_mask_ptr),
                                   C.c_void_p(int(stream)) if stream else None)
        self._resample_check(rc, "resample")

    # ---- Laplacian of Gaussian (lm_laplacian_of_gaussian_dev)
    def laplacian_of_gaussian_dev(self, d_vol_ptr, dtype_code, shape, spacing_xyz, sigma_mm, d_work_ptrs, d_out_ptr,
                                  stream=0):
        """Writes the LoG image (ITK's LaplacianRecursiveGaussianImageFilter normalised across scale, `sigma_mm` with
        spacing (x, y, z) in mm) of a C-contiguous `shape` device volume of element type `dtype_code` to the float64
        `shape` device buffer `d_out_ptr`, with the two float64 `shape` device work volumes d_work_ptrs.  ValueError for
        a refused argument or a NaN or +-inf in the volume; NativeError for the other failures."""
        n0, n1, n2 = (int(x) for x in shape)
        sp = np.array([float(s) for s in spacing_xyz], np.float64)
        if sp.shape != (3,):
            raise ValueError("laplacian_of_gaussian_dev: spacing must be (x, y, z), got %s" % (spacing_xyz,))
        w0, w1 = (C.c_void_p(int(p)) for p in d_work_ptrs)
        rc = lib().lm_laplacian_of_gaussian_dev(self._h, C.c_void_p(d_vol_ptr), int(dtype_code), n0, n1, n2, _ptr(sp),
                                                float(sigma_mm), w0, w1, C.c_void_p(d_out_ptr),
                                                C.c_void_p(int(stream)) if stream else None)
        self._resample_check(rc, "log")

    # ---- one volume over several GPUs (one engine per rank; see include/lungmask_b200.h)
    def shard_init(self, rank, world, max_slices):
        _check(lib().lm_shard_init(self._h, int(rank), int(world), int(max_slices)))
        self.shard_rank, self.shard_world = int(rank), int(world)

    def shard_export(self):
        buf = C.create_string_buffer(int(lib().lm_shard_handle_bytes()))
        _check(lib().lm_shard_export(self._h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def shard_connect(self, handles):
        """`handles`: the ranks' shard_export() results in rank order."""
        blob = b"".join(bytes(h) for h in handles)
        if len(blob) != self.shard_world * int(lib().lm_shard_handle_bytes()):
            raise ValueError("shard_connect expects %d handles" % self.shard_world)
        buf = C.create_string_buffer(blob, len(blob))
        _check(lib().lm_shard_connect(self._h, C.cast(buf, C.c_void_p)))

    def shard_labels(self):
        """(device pointer of the gathered boxes, device pointer of the gathered labels, slice capacity)"""
        b, l, cap = C.c_void_p(), C.c_void_p(), C.c_size_t(0)
        _check(lib().lm_shard_labels(self._h, C.byref(b), C.byref(l), C.byref(cap)))
        return b.value, l.value, int(cap.value)

    def apply_volume_sharded(self, slot, vol, postprocess=True, want_output=True):
        vol = _as(vol, np.int16, 3)
        S, H, W = vol.shape
        out = np.empty(vol.shape, np.uint8) if want_output else None
        _check(lib().lm_apply_volume_sharded(self._h, slot, _ptr(vol), S, H, W, 0 if postprocess else FLAG_NO_POSTPROCESS,
                                             _ptr(out) if out is not None else None))
        return out

    def apply_volume_sharded_dev(self, slot, d_vol_ptr, shape, d_out_ptr, postprocess=True):
        S, H, W = shape
        _check(lib().lm_apply_volume_sharded_dev(self._h, slot, C.c_void_p(d_vol_ptr), S, H, W,
                                                 0 if postprocess else FLAG_NO_POSTPROCESS, C.c_void_p(d_out_ptr)))

    def fuse(self, res_l, res_r):
        """mask.py:228-230 -> (fused uint8 volume before the post-processing, spare value)."""
        res_l, res_r = _as(res_l, np.uint8, 3), _as(res_r, np.uint8, 3)
        if res_l.shape != res_r.shape:
            raise ValueError("fuse: shapes differ")
        out = np.empty(res_l.shape, np.uint8)
        spare = C.c_int(0)
        S, H, W = res_l.shape
        _check(lib().lm_fuse(self._h, _ptr(res_l), _ptr(res_r), S, H, W, _ptr(out), C.byref(spare)))
        return out, int(spare.value)

    # ---- stages
    def preprocess(self, vol, out_h=NET_RES, out_w=NET_RES, clip=True):
        vol = _as(vol, np.int16, 3)
        S, H, W = vol.shape
        resized = np.empty((S, out_h, out_w), np.int16)
        boxes = np.empty((S, 4), np.int32)
        _check(lib().lm_preprocess(self._h, _ptr(vol), S, H, W, out_h, out_w, 1 if clip else 0, _ptr(resized), _ptr(boxes)))
        return resized, boxes

    def simple_bodymask(self, img):
        img = _as(img, np.int16, 2)
        out = np.empty(img.shape, np.uint8)
        _check(lib().lm_simple_bodymask(self._h, _ptr(img), img.shape[0], img.shape[1], _ptr(out)))
        return out

    def forward(self, slot, resized, return_scores=False):
        resized = _as(resized, np.int16, 3)
        S = resized.shape[0]
        if resized.shape[1:] != (NET_RES, NET_RES):
            raise ValueError("forward expects (S,256,256) slices")
        labels = np.empty((S, NET_RES, NET_RES), np.uint8)
        scores = None
        if return_scores:
            scores = np.empty((S, self.n_classes[slot], NET_RES, NET_RES), np.float32)
        _check(lib().lm_forward(self._h, slot, _ptr(resized), S, _ptr(labels), _ptr(scores) if scores is not None else None))
        return (labels, scores) if return_scores else labels

    def forward_dev(self, slot, d_resized_ptr, S, d_labels_ptr):
        ms = C.c_float(0)
        _check(lib().lm_forward_dev(self._h, slot, C.c_void_p(d_resized_ptr), S, C.c_void_p(d_labels_ptr), C.byref(ms)))
        return float(ms.value)

    def postprocess(self, labels, spare=(), skip_below=3):
        labels = _as(labels, np.uint8, 3)
        S, H, W = labels.shape
        sp = np.asarray(list(spare), dtype=np.int32)
        out = np.empty(labels.shape, np.uint8)
        _check(lib().lm_postprocess(self._h, _ptr(labels), S, H, W, _ptr(sp) if sp.size else None, int(sp.size), int(skip_below), _ptr(out)))
        return out

    def keep_largest_component(self, mask):
        mask = _as(mask, np.uint8, 3)
        out = np.empty(mask.shape, np.uint8)
        _check(lib().lm_keep_largest_component(self._h, _ptr(mask), mask.shape[0], mask.shape[1], mask.shape[2], _ptr(out)))
        return out

    def reshape_masks(self, masks, boxes, H, W):
        masks = _as(masks, np.uint8, 3)
        boxes = _as(boxes, np.int32, 2)
        S = masks.shape[0]
        out = np.empty((S, H, W), np.uint8)
        _check(lib().lm_reshape_masks(self._h, _ptr(masks), masks.shape[1], masks.shape[2], _ptr(boxes), S, H, W, _ptr(out)))
        return out

    def read_activation(self, act_id, n):
        lv, ch, sp = C.c_int(0), C.c_int(0), C.c_int(0)
        _check(lib().lm_debug_activation_info(act_id, C.byref(lv), C.byref(ch), C.byref(sp)))
        hw = NET_RES >> lv.value
        out = np.empty((n, hw, hw, ch.value), np.float32)
        _check(lib().lm_debug_read_activation(self._h, act_id, n, _ptr(out)))
        return out

    def activation_scale(self, slot, act_id):
        """The power-of-two scale activation `act_id` of weight slot `slot` is stored at (1.0 unless it was rescued)."""
        s = C.c_float(0)
        _check(lib().lm_debug_activation_scale(self._h, slot, act_id, C.byref(s)))
        return float(s.value)

    def set_option(self, key, value):
        _check(lib().lm_set_option(self._h, key.encode(), int(value)))

    def last_conv_timing(self):
        ms, n = C.c_float(0), C.c_int64(0)
        _check(lib().lm_last_conv_timing(self._h, C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)

    def last_timings(self):
        ms = (C.c_float * 7)()
        n = C.c_int64(0)
        _check(lib().lm_last_timings(self._h, ms, C.byref(n)))
        keys = ["h2d", "preprocess", "forward", "postprocess", "reshape", "d2h", "total"]
        d = {k: float(v) for k, v in zip(keys, ms)}
        d["kernel_launches"] = int(n.value)
        return d
