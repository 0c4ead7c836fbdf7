"""Host-side mirror of lungmask/mask.py for the H100 engine.

Same public names, arguments and error behaviour as the reference (`MODEL_URLS`, `get_model`,
`LMInferer`, deprecated `apply` / `apply_fused`; lungmask/mask.py:22-35,38-68,71-232,235-279), but the
work behind `LMInferer.apply` is the CUDA engine in liblungmask_b200.so.  PyTorch is used only to
read a .pth state_dict into a flat fp32 blob (lungmask_b200.h: lm_load_weights).
"""
import collections
import os
import warnings
from typing import Optional, Union

import numpy as np

from . import _native, orient
from .logger import logger

# model name -> (release URL, number of classes); lungmask/mask.py:22-35
_RELEASES = "https://github.com/JoHof/lungmask/releases/download/v0.0/"
MODEL_URLS = {
    "R231": (_RELEASES + "unet_r231-d5d2fc3d.pth", 3),
    "LTRCLobes": (_RELEASES + "unet_ltrclobes-3a07043d.pth", 6),
    "R231CovidWeb": (_RELEASES + "unet_r231covid-0de78a7e.pth", 3),
}

_CH = [64, 128, 256, 512, 1024]


def _conv3x3_prefixes():
    """The 18 Conv3x3+BN pairs in execution order (resunet.py:58-67): (conv prefix, bn prefix)."""
    out = []
    for i in range(5):
        out += [(f"down_path.{i}.block.0", f"down_path.{i}.block.2"), (f"down_path.{i}.block.3", f"down_path.{i}.block.5")]
    for j in range(4):
        p = f"up_path.{j}.conv_block.block"
        out += [(p + ".0", p + ".2"), (p + ".3", p + ".5")]
    return out


class NativeModel:
    """What `get_model` returns here: the live tensors of a reference state_dict flattened in the
    order lm_load_weights expects, plus the class count.  The dead `residual_*` tensors and the BN
    `num_batches_tracked` counters of the reference layout are validated for presence and dropped."""

    def __init__(self, state_dict):
        import torch

        def t(key, shape=None):
            if key not in state_dict:
                raise KeyError("state_dict is missing %r (not a lungmask U-Net checkpoint?)" % key)
            a = state_dict[key].detach().to(torch.float32).cpu().contiguous().numpy()
            if shape is not None and tuple(a.shape) != tuple(shape):
                raise ValueError("%s has shape %s, expected %s" % (key, tuple(a.shape), tuple(shape)))
            return a.ravel()

        # mask.py:56: the class count is the length of the LAST tensor of the state_dict
        self.n_classes = int(len(list(state_dict.values())[-1]))
        K = self.n_classes
        parts = []
        cin = 1
        chans = []  # (cin, cout) for the 18 convs
        for i in range(5):
            chans += [(cin, _CH[i]), (_CH[i], _CH[i])]
            cin = _CH[i]
        for j in range(4):
            c = _CH[3 - j]
            chans += [(2 * c, c), (c, c)]
        for (conv, bn), (ci, co) in zip(_conv3x3_prefixes(), chans):
            parts += [t(conv + ".weight", (co, ci, 3, 3)), t(conv + ".bias", (co,)), t(bn + ".weight", (co,)),
                      t(bn + ".bias", (co,)), t(bn + ".running_mean", (co,)), t(bn + ".running_var", (co,))]
        for j in range(4):
            c = _CH[3 - j]
            parts += [t(f"up_path.{j}.up.1.weight", (c, 2 * c, 1, 1)), t(f"up_path.{j}.up.1.bias", (c,))]
        parts += [t("last.weight", (K, 64, 1, 1)), t("last.bias", (K,))]
        self.blob = np.ascontiguousarray(np.concatenate(parts), dtype=np.float32)


def get_model(modelname: str, modelpath: Optional[str] = None) -> NativeModel:
    """lungmask/mask.py:38-68.  `modelpath` given: torch.load of that file; otherwise the released
    weights are fetched through torch.hub (needs network).  The class count always comes from the
    file, never from `modelname`."""
    import torch

    if modelpath is None:
        url, _ = MODEL_URLS[modelname]
        state_dict = torch.hub.load_state_dict_from_url(url, progress=True, map_location=torch.device("cpu"))
    else:
        state_dict = torch.load(modelpath, map_location=torch.device("cpu"))
    return NativeModel(state_dict)


def _to_int16_volume(image: np.ndarray) -> np.ndarray:
    """Integer volumes.  Integers of any width give the same result as the reference because it clips to [-1024, 600]
    before resampling (utils.py:45) and thresholds at -500 HU, so they are clipped into int16 here."""
    if image.ndim != 3:
        raise ValueError("expected a (slices, H, W) volume, got shape %s" % (image.shape,))
    if image.dtype == np.int16:
        return np.ascontiguousarray(image)
    if np.issubdtype(image.dtype, np.integer) or image.dtype == bool:
        return np.clip(image, -1024, 600).astype(np.int16)
    raise TypeError("not an integer volume: %s" % image.dtype)


def _to_engine_volume(image: np.ndarray) -> np.ndarray:
    """The array the engine receives: int16 for integer volumes; float32 / float64 volumes keep their dtype, as they do
    in the reference (utils.preprocess clips and resamples in the input dtype and mask.py:167-168 normalises in it; the
    engine has a float path for exactly that).  Other float widths are widened to float32 (the reference would compute
    in float16 / longdouble there: documented deviation)."""
    if image.ndim != 3:
        raise ValueError("expected a (slices, H, W) volume, got shape %s" % (image.shape,))
    if image.dtype in (np.float32, np.float64):
        return np.ascontiguousarray(image)
    if np.issubdtype(image.dtype, np.floating):
        logger.warning("volume dtype %s is computed as float32", image.dtype)
        return np.ascontiguousarray(image, dtype=np.float32)
    return _to_int16_volume(image)


def _is_tensor(image) -> bool:
    import torch
    return isinstance(image, torch.Tensor)


def _tensor_dtype_code(t) -> int:
    """LM_DTYPE_* of lm_apply_dev for a tensor's dtype; TypeError for the dtypes the engine does not read."""
    import torch
    codes = {torch.bool: _native.DTYPE_U8, torch.uint8: _native.DTYPE_U8, torch.int8: _native.DTYPE_I8,
             torch.int16: _native.DTYPE_I16, torch.int32: _native.DTYPE_I32, torch.int64: _native.DTYPE_I64,
             torch.float16: _native.DTYPE_F16, torch.bfloat16: _native.DTYPE_BF16, torch.float32: _native.DTYPE_F32,
             torch.float64: _native.DTYPE_F64}
    if t.dtype not in codes:
        raise TypeError("volume tensor dtype %s is not supported: use bool, uint8, a signed integer type, float16, bfloat16, "
                        "float32 or float64" % t.dtype)
    return codes[t.dtype]


# numpy dtype -> LM_DTYPE_* of a host volume of the analysis calls
_HOST_DTYPE_CODES = {np.dtype(bool): _native.DTYPE_U8, np.dtype(np.uint8): _native.DTYPE_U8, np.dtype(np.int8): _native.DTYPE_I8,
                     np.dtype(np.int16): _native.DTYPE_I16, np.dtype(np.int32): _native.DTYPE_I32,
                     np.dtype(np.int64): _native.DTYPE_I64, np.dtype(np.float16): _native.DTYPE_F16,
                     np.dtype(np.float32): _native.DTYPE_F32, np.dtype(np.float64): _native.DTYPE_F64}


def _host_volume(vol, what):
    """(C-contiguous array, LM_DTYPE_* code) of a host volume of the analysis calls: uint16 / uint32 widened to int32 / int64
    without loss; TypeError for the dtypes the engine does not read."""
    if vol.dtype in (np.uint16, np.uint32):
        vol = vol.astype(np.int32 if vol.dtype == np.uint16 else np.int64)
    if vol.dtype not in _HOST_DTYPE_CODES:
        raise TypeError("%s: volume dtype %s is not supported" % (what, vol.dtype))
    return np.ascontiguousarray(vol), _HOST_DTYPE_CODES[vol.dtype]


# What LMInferer._stage hands an analysis call: the volume (None for a mask alone), its LM_DTYPE_* code and the uint8 mask
# as contiguous CUDA tensors on the engine's device, the caller's cudaStream_t, the spacing (x, y, z) or None, the
# orientation code of the arrays, and back(t): a result tensor of the mask's shape in the type the mask came as.
_Staged = collections.namedtuple("_Staged", "vol dtype mask stream spacing orientation back")


class LMInferer:
    def __init__(
        self,
        modelname: str = "R231",
        modelpath: Optional[str] = None,
        fillmodel: Optional[str] = None,
        fillmodel_path: Optional[str] = None,
        force_cpu: bool = False,
        batch_size: int = 20,
        volume_postprocessing: bool = True,
        tqdm_disable: bool = False,
        device: Optional[int] = None,
        wave_slices: Optional[int] = None,
    ):
        """Same arguments as the reference (lungmask/mask.py:72-82) plus `device` (CUDA ordinal, default
        LOCAL_RANK or 0) and `wave_slices`.  The reference's `batch_size` only bounds memory (slices are
        independent, mask.py:172-187; the engine is batch-invariant, tests/test_gpu_forward.py); the engine
        runs the forward in waves of `wave_slices` slices, default 33 when batch_size >= 20 because
        33 x 16 tiles = 4 x 132 SMs fills every level of the U-Net with whole waves of CTAs (about 5 GB of
        activations), else batch_size."""
        assert modelname in MODEL_URLS, "Modelname not found. Please choose from: {}".format(MODEL_URLS.keys())
        if fillmodel is not None:
            assert fillmodel in MODEL_URLS, "Modelname not found. Please choose from: {}".format(MODEL_URLS.keys())
        if modelpath is not None:  # a path overrides the name (mask.py:104-107)
            modelname = os.path.basename(modelpath)
        if fillmodel_path is not None:
            fillmodel = os.path.basename(fillmodel_path)
        if force_cpu:
            raise RuntimeError("lungmask_b200 is an H100 (sm_90a) engine and has no CPU path; "
                               "use the reference package for force_cpu=True")
        self.fillmodel = fillmodel
        self.modelname = modelname
        self.force_cpu = force_cpu
        self.batch_size = batch_size
        self.volume_postprocessing = volume_postprocessing
        self.tqdm_disable = tqdm_disable
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0"))
        self.device = device

        self.model = get_model(self.modelname, modelpath)
        if wave_slices is None:
            wave_slices = 33 if batch_size >= 20 else batch_size
            if batch_size >= 20 and os.environ.get("LM_WAVE_SLICES"):   # measurement hook: 66 = eight CTA rounds per level
                wave_slices = max(1, min(1024, int(os.environ["LM_WAVE_SLICES"])))
        self.wave_slices = wave_slices
        self.engine = _native.Engine(device=device, batch_capacity=wave_slices)
        self.engine.load_weights(0, self.model.blob, self.model.n_classes)
        self.fillmodelm = None
        if self.fillmodel is not None:
            self.fillmodelm = get_model(self.fillmodel, fillmodel_path)
            self.engine.load_weights(1, self.fillmodelm.blob, self.fillmodelm.n_classes)

    # -- SimpleITK inputs are oriented to LPS first and back afterwards (mask.py:157-164,204-208): here that is an
    #    axis permutation + flips done by the engine on the device (lungmask_b200/orient.py, lm_apply_volume_oriented)
    @staticmethod
    def _sitk():
        try:
            import SimpleITK as sitk
            return sitk
        except Exception:
            return None

    def _log_fusion(self):
        logger.info(f"Apply: {self.modelname}")
        logger.info(f"Apply: {self.fillmodel}")
        logger.info("Fusing results... this may take up to several minutes!")

    def _run(self, volume: np.ndarray, code: str = "LPS") -> np.ndarray:
        vol = _to_engine_volume(volume)
        fused = self.fillmodel is not None
        if vol.dtype != np.int16 and code != "LPS" and fused:
            # the fusion runs in the native orientation (mask.py:225-232): the engine's device path does the re-orientation,
            # so the volume goes through a CUDA tensor on the engine's device
            import torch
            src = torch.from_numpy(vol if vol.flags.writeable else vol.copy()).to(torch.device("cuda", self.engine.device))
            return self._run_tensor(src, code).cpu().numpy()
        if fused:
            self._log_fusion()
        if vol.dtype != np.int16:   # float volume
            if code != "LPS":       # re-orient on the host (rare: float + non-LPS); the integer path does it on the device
                res = self.engine.apply_volume_float(0, orient.to_lps(vol, code), slot_fill=-1,
                                                     postprocess=self.volume_postprocessing)
                return orient.from_lps(res, code)
            return self.engine.apply_volume_float(0, vol, slot_fill=1 if fused else -1, postprocess=self.volume_postprocessing)
        if code == "LPS":
            if not fused:
                return self.engine.apply_volume(0, vol, postprocess=self.volume_postprocessing)
            return self.engine.apply_fused(0, 1, vol, postprocess=self.volume_postprocessing)
        perm, flip = orient.array_transform_to_lps(code)
        return self.engine.apply_volume_oriented(0, vol, perm, flip, slot_fill=1 if fused else -1,
                                                 postprocess=self.volume_postprocessing)

    def _run_tensor(self, t, code: str = "LPS", with_probs: bool = False):
        """A torch.Tensor volume (slices, H, W).  A CUDA tensor on the engine's device is segmented where it lies
        (lm_apply_dev, ordered after the work queued on the current stream): the uint8 mask (and the float32 probabilities)
        come back as tensors on that device.  A CPU tensor takes the numpy path and gets CPU tensors back."""
        import torch
        if t.dim() != 3:
            raise ValueError("expected a (slices, H, W) volume, got shape %s" % (tuple(t.shape),))
        dtype_code = _tensor_dtype_code(t)
        if t.device.type not in ("cpu", "cuda"):
            raise ValueError("the volume tensor is on %s: give a CPU tensor or a CUDA tensor on cuda:%d" % (t.device, self.engine.device))
        t = t.detach()
        if not t.is_cuda:
            if t.dtype == torch.bfloat16:   # numpy has no bfloat16: widen here, with the warning of the float16 path
                logger.warning("volume dtype %s is computed as float32", t.dtype)
                t = t.float()
            a = t.numpy()
            if with_probs:
                mask, probs = self._probabilities(a, code)
                return torch.from_numpy(mask), torch.from_numpy(probs)
            return torch.from_numpy(self._run(a, code))
        if t.device.index != self.engine.device:
            raise ValueError("the volume tensor is on %s, the engine on cuda:%d" % (t.device, self.engine.device))
        if t.dtype in (torch.float16, torch.bfloat16):
            logger.warning("volume dtype %s is computed as float32", t.dtype)
        if not t.is_contiguous():
            t = t.contiguous()
        fused = self.fillmodel is not None
        if fused:
            self._log_fusion()
        perm, flip = (None, None) if code == "LPS" else orient.array_transform_to_lps(code)
        out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
        probs = None
        if with_probs:
            probs = torch.empty((self.engine.n_classes[0],) + tuple(t.shape), dtype=torch.float32, device=t.device)
        self.engine.apply_dev(0, t.data_ptr(), dtype_code, t.shape, out.data_ptr(), perm, flip, slot_fill=1 if fused else -1,
                              d_probs_ptr=probs.data_ptr() if probs is not None else None,
                              postprocess=self.volume_postprocessing, stream=torch.cuda.current_stream(t.device).cuda_stream)
        return (out, probs) if with_probs else out

    def apply_oriented(self, array, direction):
        """What `apply(sitk_image)` does, for callers without SimpleITK: `array` = sitk.GetArrayFromImage(image)
        (axes z, y, x) as a numpy array or a torch.Tensor, `direction` = image.GetDirection() (9 direction cosines).  The
        mask comes back in the array's own orientation (mask.py:157-164,204-208), as a tensor for a tensor (see `apply`)."""
        code = orient.orientation_from_direction(direction)
        if _is_tensor(array):
            return self._run_tensor(array, code)
        return self._run(array, code)

    def _array_and_orientation(self, image, caller: str = "apply"):
        """(array (z, y, x), orientation code) of what `apply` accepts: a numpy array is taken as LPS; a
        lungmask_b200.io.Volume or a SimpleITK image carries its direction cosines."""
        if isinstance(image, np.ndarray):
            return image, "LPS"
        from .io import Volume
        if isinstance(image, Volume):       # what lungmask_b200.io.load_input_image returns
            return image.array, orient.orientation_from_direction(image.GetDirection())
        sitk = self._sitk()
        if sitk is None or not isinstance(image, sitk.Image):
            raise TypeError("%s() expects a numpy array, a SimpleITK image or a lungmask_b200.io.Volume" % caller)
        return sitk.GetArrayFromImage(image), orient.orientation_from_direction(image.GetDirection())

    def apply(self, image):
        """Segments a volume: numpy (slices, H, W), sitk.Image or lungmask_b200.io.Volume -> uint8 labels of the same shape
        (lungmask/mask.py:212-232).  The input is not modified.

        A torch.Tensor (slices, H, W) is taken as LPS, like a numpy array.  A CUDA tensor on the engine's device never
        leaves the GPU: the engine waits for the work queued on the current stream, reads the tensor in place (int16,
        float32, float64) or converts it on the device (bool and other integers are clipped to [-1024, 600], float16 /
        bfloat16 are widened to float32), and returns a uint8 tensor on that device, complete when the call returns.  A CPU
        tensor gives what its numpy array gives, as a CPU tensor."""
        if _is_tensor(image):
            return self._run_tensor(image)
        return self._run(*self._array_and_orientation(image))

    def _probabilities(self, array, code):
        vol = _to_engine_volume(array)
        perm, flip = (None, None) if code == "LPS" else orient.array_transform_to_lps(code)
        return self.engine.apply_volume_probs(0, vol, perm, flip, postprocess=self.volume_postprocessing)

    def apply_with_probabilities(self, image):
        """The mask and the per-class probabilities of the model from one forward pass: image as for `apply` ->
        (mask, probabilities).

        `mask` is bit-identical to `apply(image)`, `volume_postprocessing` included.  `probabilities` is float32 of shape
        (K, *mask.shape), in the input's own geometry and orientation: probabilities[k] = exp of the network's
        log-softmax score of class k (what the reference's `inferer.model(x)` returns), taken from the network pixel
        that the mask's order-0 resampling (utils.reshape_mask) puts at that voxel.  Voxels outside the slice's body
        crop box are background with probability 1.  The probabilities are the network's output BEFORE
        post-processing; with volume_postprocessing=False, their argmax is the mask.  Needs K * mask.size * 4 bytes on
        the device and on the host.  Not defined for a fill model (the reference's fusion has no probabilities).

        For a CUDA tensor on the engine's device (see `apply`) both come back as tensors on that device, bit-identical to
        the numpy results, with no copy to the host."""
        if self.fillmodel is not None:
            raise ValueError("apply_with_probabilities: the fusion with a fill model (%s) has no class probabilities; "
                             "use an LMInferer without fillmodel" % self.fillmodel)
        if _is_tensor(image):
            return self._run_tensor(image, with_probs=True)
        return self._probabilities(*self._array_and_orientation(image, "apply_with_probabilities"))

    def statistics(self, image, mask, spacing=None, percentiles=(15.0,), thresholds=(-950,)):
        """Per-label volume and HU statistics of `image` under `mask` (e.g. the mask `apply(image)` returned) ->
        lungmask_b200.statistics.LabelStatistics: a row for every label value in the mask and every label 1..K-1 of the
        model (absent ones with 0 voxels), then "lung", the union of all labels.  Each row holds the voxel count, the
        volume in mL (when a spacing is known), the NaN count, mean / std / min / max HU, numpy.percentile of the values
        for each of `percentiles` (bit-identical) and the fraction of the values below each integer HU of `thresholds`.
        The defaults are Perc15 and LAA-950.

        `image`: what `apply` accepts, with `mask` (uint8 or bool) of the same shape in the same array orientation; the
        values are taken as they are (not clipped).  A Volume or SimpleITK image supplies its spacing (x, y, z) in mm
        unless `spacing` is given.  A CUDA tensor with a CUDA mask tensor on the engine's device is read in place, ordered
        after the work queued on the current stream; numpy arrays and CPU tensors are uploaded.  Both inputs are left
        unchanged."""
        from . import statistics as st
        q, t = st.check_arguments(percentiles, thresholds)
        s = self._stage("statistics", image, mask, spacing)
        res = self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), s.mask.shape, q, t, stream=s.stream)
        labels = set(np.nonzero(res["voxels"][1:256])[0] + 1) | set(range(1, self.engine.n_classes[0]))
        return st.from_native(res, labels, self.modelname, s.spacing, q, t)

    def laa_clusters(self, image, mask, threshold=-950, connectivity=6, spacing=None, min_cluster_voxels=1):
        """Size distributions of the connected clusters of low-attenuation voxels (mask > 0 and value < `threshold` HU)
        per label and for the whole lung -> lungmask_b200.clusters.LaaClusters, with the rows of `statistics`: every
        label value in the mask and every label 1..K-1 of the model, then "lung".  A label's clusters never cross its
        boundary; the "lung" row labels all LAA voxels together, so a cluster there may span two lobes.

        Each row holds the LAA voxel count and volume (mL, when a spacing is known), the number of clusters, the largest
        cluster (voxels and mL), the exact distribution as `sizes` / `counts` arrays (ascending sizes, int64), and D,
        the exponent of the power law of the cumulative size distribution (Mishima et al., PNAS 1999): minus the
        least-squares slope of log10 Y(s) on log10 s, one point per distinct size s >= `min_cluster_voxels`, Y(s) = the
        number of clusters of s voxels or more; NaN with fewer than two points.  That is one convention among several
        (binning, size cut-offs, fit ranges differ between studies); the raw pairs are there for the others.

        `connectivity`: 6 (faces, scipy.ndimage.label's default), 26 (full, as the post-processing) or 4 (faces within a
        slice: per-slice 2-D clusters as in the original 2-D analysis).  `threshold`: an integer HU in [-1024, 3072],
        compared in the volume's dtype (not clipped; NaN is never LAA).  `image`, `mask` and `spacing` as for
        `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the spacing), CPU tensors, or CUDA tensors
        on the engine's device read in place after the work queued on the current stream."""
        from . import clusters as cl
        threshold, connectivity, min_cluster_voxels = cl.check_arguments(threshold, connectivity, min_cluster_voxels)
        s = self._stage("laa_clusters", image, mask, spacing)
        res = self.engine.laa_clusters_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), s.mask.shape, threshold, connectivity,
                                           stream=s.stream)
        labels = self._mask_labels(s.mask, s.stream) | set(range(1, self.engine.n_classes[0]))
        return cl.from_native(res, labels, self.modelname, s.spacing, threshold, connectivity, min_cluster_voxels)

    def surface_distance(self, mask, spacing):
        """The distance in mm from every voxel with mask > 0 to the nearest voxel with mask == 0 -> float32 of the mask's
        shape: 0 outside the mask, +inf when the mask has no zero voxel.  The surface is that of the union of all labels,
        so fissures between lobes are interior.  Voxels outside the array are not background (as in
        scipy.ndimage.distance_transform_edt): a lung cut off by the first or last slice has no surface there.

        `spacing`: the voxel size along each ARRAY axis, (s0, s1, s2) in mm, as scipy's `sampling` - for a Volume or
        SimpleITK image that is GetSpacing()[::-1].  The exact Euclidean distance is computed in float64 on the GPU and
        rounded once: np.float32(scipy.ndimage.distance_transform_edt(mask > 0, sampling=spacing)) bit for bit when the
        squared distances are exact in float64 (dyadic spacings such as 0.703125 or 1.25), else within 1 float32 ulp.

        `mask`: (S, H, W) uint8 or bool, numpy or a torch tensor.  A CUDA tensor on the engine's device is read in place
        after the work queued on the current stream and the result is a float32 CUDA tensor there; a CPU tensor gives a
        CPU tensor.  The mask is left unchanged."""
        import torch
        sp = tuple(float(s) for s in np.asarray(spacing, dtype=np.float64).reshape(-1))
        if len(sp) != 3 or not all(np.isfinite(s) and s > 0 for s in sp):
            raise ValueError("surface_distance: spacing must be 3 finite positive sizes (s0, s1, s2) in mm, got %s" % (spacing,))
        s = self._stage("surface_distance", None, mask, mask_only=True)
        out = torch.empty(tuple(s.mask.shape), dtype=torch.float32, device=s.mask.device)
        self.engine.surface_distance_dev(s.mask.data_ptr(), s.mask.shape, sp, out.data_ptr(), stream=s.stream)
        return s.back(out)

    def regional_statistics(self, image, mask, spacing=None, zones=3, zone_by="volume", shells_mm=(10.0,),
                            percentiles=(15.0,), thresholds=(-950,)):
        """Statistics of `image` under `mask` by craniocaudal zone and by depth below the lung surface ->
        lungmask_b200.regions.RegionalStatistics.  The rows of `statistics` (every label value in the mask, every label
        1..K-1 of the model, then "lung") are each split into `zones` craniocaudal zones and into the depth shells of
        `shells_mm`; every zone or shell row holds the full statistics.LabelRow of its voxels (see `statistics`).

        Zones are whole planes along the craniocaudal array axis: axis 0, superior at the high index, for numpy arrays
        and tensors (LPS, as in `apply`); for a Volume or SimpleITK image the axis its orientation names S or I.  Zone 0
        is the most superior; every row gets its own boundaries.  zone_by="volume" splits each row's planes at equal
        shares of its voxels (a plane goes to the zone of the midpoint of its share), "height" at equal shares of its
        first..last plane; see regions.zone_of_planes.  With 3 zones they are named upper / middle / lower.  Each zone row
        reports its plane range in array indices, and the result holds every row's voxels per plane (the profile).

        Shells: with shells_mm = (b_1, ..., b_m) strictly increasing in mm, shell j holds the voxels with
        b_j <= depth < b_{j+1} (b_0 = 0, b_{m+1} = inf) where depth = `surface_distance` (float32, compared with the
        bounds as float32).  Shell 0 is the rind.  Shells need the spacing; shells_mm=() skips them.

        `image`, `mask` and `spacing` (x, y, z) mm as for `statistics`: numpy arrays (the image is uploaded once), a
        Volume or SimpleITK image (which supplies the spacing), CPU tensors, or CUDA tensors on the engine's device read in
        place after the work queued on the current stream.  The per-label region map gives each (label, zone) and
        (label, shell) its own uint8 code, so labels x zones and labels x shells must stay at or below 255."""
        import torch
        from . import regions as rg
        zones, zone_by, shells_mm, q, t = rg.check_arguments(zones, zone_by, shells_mm, percentiles, thresholds)
        s = self._stage("regional_statistics", image, mask, spacing)
        if shells_mm and s.spacing is None:
            raise ValueError("regional_statistics: depth shells need the voxel spacing; pass spacing=(x, y, z) in mm, or "
                             "shells_mm=() for zones only")
        axis, superior_high = rg.craniocaudal_axis(s.orientation)
        m, shape = s.mask, tuple(s.mask.shape)
        counts = self.engine.plane_label_counts_dev(m.data_ptr(), shape, axis, stream=s.stream)
        present = [int(x) for x in np.flatnonzero(counts[:, 1:256].sum(axis=0)) + 1]
        rg.check_code_budget(present, zones, "zones")
        if shells_mm:
            rg.check_code_budget(present, len(shells_mm) + 1, "shells")
        label_zones = {l: rg.zone_of_planes(counts[:, l], zones, zone_by, superior_high) for l in present}
        lung_zones = rg.zone_of_planes(counts[:, 256], zones, zone_by, superior_high)
        region = torch.empty(shape, dtype=torch.uint8, device=m.device)

        def stats_of(lut, **kw):
            self.engine.region_map_dev(m.data_ptr(), shape, lut, region.data_ptr(), stream=s.stream, **kw)
            return self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, region.data_ptr(), shape, q, t, stream=s.stream)

        lut, lung_lut = rg.zone_luts(present, label_zones, lung_zones, zones)
        zone, zone_lung = stats_of(lut, axis=axis), stats_of(lung_lut, axis=axis)
        shell = shell_lung = None
        if shells_mm:
            dist = torch.empty(shape, dtype=torch.float32, device=m.device)
            self.engine.surface_distance_dev(m.data_ptr(), shape, s.spacing[::-1], dist.data_ptr(), stream=s.stream)
            lut, lung_lut = rg.shell_luts(present, len(shells_mm) + 1)
            kw = dict(d_dist_ptr=dist.data_ptr(), bounds=shells_mm)
            shell, shell_lung = stats_of(lut, **kw), stats_of(lung_lut, **kw)
        labels = sorted(set(present) | set(range(1, self.engine.n_classes[0])))
        return rg.build(labels, present, self.modelname, s.spacing, counts, axis, superior_high, zones, zone_by, shells_mm, q, t,
                        label_zones, lung_zones, zone, zone_lung, shell, shell_lung)

    def texture(self, image, mask, bin_width=25, spacing=None, classes=("glcm", "glszm"), gldm_alpha=0, distances=(1,),
                force2d=False, force2d_dimension=0, weighting_norm=None):
        """Grey-level texture features of `image` under `mask` -> lungmask_b200.texture.TextureFeatures, with the rows
        of `statistics`: every label value in the mask and every label 1..K-1 of the model (absent ones with 0 voxels and
        NaN features), then "lung" (mask > 0).  A row's ROI is its voxels with a non-NaN value, read in the volume's dtype
        (float16 / bfloat16 as float32); a non-finite value in an ROI is a ValueError.

        Each row is discretised with the fixed `bin_width` (a positive integer, PyRadiomics' binWidth): low = bw *
        floor(min / bw), level(x) = floor((floor(x) - low) / bw) + 1, Ng = the level of the row's maximum; more than 255
        levels is a ValueError before any texture kernel runs.  GLCM: the symmetric co-occurrence matrices of the 13
        directions of the 26-neighbourhood at distance 1 voxel (spacing is not used), a pair counted only when both voxels
        are in the row (so a pair across a lobe boundary counts in "lung" only); the features are averaged over the
        directions with pairs.  GLSZM: the 26-connected zones of equal level.  Each row holds the features (dicts keyed by
        the PyRadiomics names of texture.GLCM_FEATURES / GLSZM_FEATURES) and the exact matrices: the pair counts
        `glcm_counts` (13, Ng (Ng + 1) / 2) and the (level, size, count) `zones`.

        `classes` is a non-empty collection of the names "glcm", "glszm", "glrlm", "gldm" and "ngtdm", in any order; only
        those are computed, and only their keys appear in to_dict() and the writers.  GLRLM: the maximal runs of equal
        level along the 13 directions, features averaged over the directions; `glrlm_runs` holds the (direction, level,
        length, count) rows.  GLDM: per voxel the number c of its 26 neighbours in the row within `gldm_alpha` levels (a
        non-negative integer, PyRadiomics' gldm_a), dependence size c + 1; `gldm_counts` (Ng, 27).  NGTDM: per voxel the
        number W of its neighbours in the row and the sum S of their levels; `ngtdm_counts` N(i, W) and `ngtdm_sums`
        A(i, W) = sum |W i - S|, (Ng, 27).  A bad `classes` or `gldm_alpha` raises before any kernel runs.

        PyRadiomics' neighbourhood settings (DESIGN §4.18; the defaults give the matrices above): `distances`, a
        collection of integers 1..3, and `force2d` with `force2d_dimension` (0, 1 or 2, the axis normal to the planes)
        set the offsets O of texture.offsets.  GLCM then has one matrix per offset, `glcm_counts` (|O|, T); GLDM and
        NGTDM use the K = 2 |O| neighbours v +- o, matrices (Ng, K + 1).  GLSZM ignores `distances` and with force2d
        takes zones 8-connected within the planes; GLRLM ignores `distances` and with force2d uses the 4 in-plane
        directions of the 13 (`glrlm_runs` directions index texture.Settings.run_offsets()).  `weighting_norm` ("manhattan",
        "euclidean", "infinity", "no_weighting" or None) merges the GLCM and GLRLM matrices with the weights of
        texture.weights over the spacing before the features are computed once; a norm other than "no_weighting" needs
        a spacing.  Bad settings raise before any kernel runs.

        `image`, `mask` and `spacing` as for `statistics`: numpy arrays, a Volume or SimpleITK image, CPU tensors, or CUDA
        tensors on the engine's device read in place after the work queued on the current stream; both are left
        unchanged."""
        import torch
        from . import texture as tx
        from .statistics import label_name
        bw = tx.check_arguments(bin_width)
        classes = tx.check_classes(classes)
        alpha = tx.check_alpha(gldm_alpha)
        settings = tx.check_settings(distances, force2d, force2d_dimension, weighting_norm)
        s = self._stage("texture", image, mask, spacing)
        tx.check_weighting_spacing(settings, s.spacing)
        shape = tuple(s.mask.shape)
        default = settings.default_neighbourhood()
        offs = settings.offsets()
        axis = settings.force2d_dimension
        glcm_w = glrlm_w = None
        if settings.weighting_norm is not None:
            glcm_w = tx.weights(offs, settings.weighting_norm, s.spacing)
            glrlm_w = tx.weights(settings.run_offsets(), settings.weighting_norm, s.spacing)
        run_rows = [tx.OFFSETS.index(o) for o in settings.run_offsets()]
        st = self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, (), (), stream=s.stream)
        present = set(int(x) for x in np.nonzero(st["voxels"][1:256])[0] + 1)
        rows = sorted(present | set(range(1, self.engine.n_classes[0]))) + [256]
        names = {r: tx.UNION if r == 256 else label_name(self.modelname, r) for r in rows}
        plan = {}   # every row's discretisation first: a refused row stops the call before any texture kernel
        for r in rows:
            n = int(st["voxels"][r] - st["nan_voxels"][r])
            if n:
                plan[r] = (n,) + tx.discretisation(float(st["moments"][r][2]), float(st["moments"][r][3]), bw,
                                                   "row %s (%s)" % ("lung" if r == 256 else r, names[r]))
        out = []
        levels = torch.empty(shape, dtype=torch.uint8, device=s.mask.device) if plan else None
        for r in rows:
            if r not in plan:
                out.append(tx.build_row(r, names[r], 0, bw, classes=classes, columns=2 * len(offs) + 1))
                continue
            n, low, ng = plan[r]
            self.engine.texture_levels_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, r, low, bw, ng,
                                           levels.data_ptr(), stream=s.stream)
            U = zones = runs = neighbours = None
            if "glcm" in classes:
                U = (self.engine.glcm_dev(levels.data_ptr(), shape, ng, stream=s.stream) if default else
                     self.engine.glcm_offsets_dev(levels.data_ptr(), shape, ng, offs, stream=s.stream))
            if "glszm" in classes:
                zones = tx.zones_from_native(
                    self.engine.zone_sizes_dev(levels.data_ptr(), shape, stream=s.stream) if axis is None else
                    self.engine.zone_sizes_plane_dev(levels.data_ptr(), shape, axis, stream=s.stream))
            if "glrlm" in classes:
                runs = self.engine.glrlm_dev(levels.data_ptr(), shape, ng, stream=s.stream)
                if axis is not None:
                    runs = runs[run_rows]
            if "gldm" in classes or "ngtdm" in classes:
                # |level difference| <= ng - 1 always, so a larger alpha counts the same neighbours
                a = min(alpha, tx.MAX_LEVELS)
                neighbours = (self.engine.neighbour_counts_dev(levels.data_ptr(), shape, ng, a, stream=s.stream) if default
                              else self.engine.neighbour_offsets_dev(levels.data_ptr(), shape, ng, offs, a, stream=s.stream))
            out.append(tx.build_row(r, names[r], n, bw, low, ng, U, zones, classes, runs, neighbours, glcm_w, glrlm_w,
                                    2 * len(offs) + 1))
        return tx.TextureFeatures(s.spacing, bw, out, classes, alpha, settings)

    def first_order(self, image, mask, bin_width=25, spacing=None, voxel_array_shift=0):
        """PyRadiomics' 18 default first-order features of `image` under `mask` -> lungmask_b200.first_order.
        FirstOrderFeatures, with the rows of `statistics`: every label value in the mask and every label 1..K-1 of the
        model (absent ones with 0 voxels and NaN features), then "lung" (mask > 0).  A row's ROI is its voxels with a
        non-NaN value, read in the volume's dtype (float16 / bfloat16 as float32); a non-finite value in an ROI is a
        ValueError.

        The features (first_order.FIRST_ORDER_FEATURES) are the percentiles, Minimum, Maximum and Range of numpy.percentile
        (bit-identical; Median is the 50th percentile), Mean, Variance, Skewness and Kurtosis (m4 / m2^2, not excess; both
        0 when m2 = 0), MeanAbsoluteDeviation, RobustMeanAbsoluteDeviation (over P10 <= x <= P90), Energy = sum (x + c)^2
        with c = `voxel_array_shift` (an integer, PyRadiomics' voxelArrayShift), TotalEnergy = Energy x the voxel volume
        in mm^3 (NaN without a spacing), RootMeanSquared, and Entropy and Uniformity of the level histogram of the
        fixed `bin_width` discretisation of `texture` (more than 255 levels in any row is a ValueError before any
        first-order kernel runs).  Integer rows that span fewer than 2^20 values are summed exactly: their features are
        reproducible bit for bit (`exact` on the row).  Each row keeps the level histogram, the power and split sums and
        the percentiles its features come from.

        `image`, `mask` and `spacing` as for `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the
        spacing), CPU tensors, or CUDA tensors on the engine's device read in place after the work queued on the current
        stream; both are left unchanged."""
        from . import first_order as fo
        from . import texture as tx
        from .statistics import label_name
        bw = tx.check_arguments(bin_width)
        shift = fo.check_shift(voxel_array_shift)
        s = self._stage("first_order", image, mask, spacing)
        shape = tuple(s.mask.shape)
        st = self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, fo.PERCENTILES, (),
                                         stream=s.stream)
        present = set(int(x) for x in np.nonzero(st["voxels"][1:256])[0] + 1)
        rows = sorted(present | set(range(1, self.engine.n_classes[0]))) + [256]
        names = {r: fo.UNION if r == 256 else label_name(self.modelname, r) for r in rows}
        integer = s.dtype in (_native.DTYPE_U8, _native.DTYPE_I8, _native.DTYPE_I16, _native.DTYPE_I32, _native.DTYPE_I64)
        plan = {}   # every row's plan first: a refused row stops the call before any first-order kernel
        for r in rows:
            n = int(st["voxels"][r] - st["nan_voxels"][r])
            if n:
                m = st["moments"][r]
                plan[r] = fo.plan_row(n, float(m[2]), float(m[3]), float(m[0]), st["percentile"][r], bw, integer,
                                      "row %s (%s)" % ("lung" if r == 256 else r, names[r]))
        if not plan:
            return fo.FirstOrderFeatures(s.spacing, bw, shift, [fo.build_row(r, names[r], bw) for r in rows])
        mode = np.zeros(257, np.int32)
        low, base, split, split_b = (np.zeros(257, np.int64) for _ in range(4))
        n_levels = np.zeros(257, np.int32)
        centre, centre_b, band_lo, band_hi = (np.zeros(257, np.float64) for _ in range(4))
        for r, p in plan.items():
            mode[r] = fo.MODE_EXACT if p.exact else fo.MODE_FLOAT
            low[r], n_levels[r], base[r], centre[r] = p.low, p.n_levels, p.base, p.mean
            band_lo[r], band_hi[r] = p.percentiles[0], p.percentiles[4]
        a = self.engine.first_order_sums_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, bw, mode, low, n_levels, base,
                                             centre, band_lo, band_hi, stream=s.stream)
        sums = {}
        for r, p in plan.items():
            if p.exact:
                w = fo.int_sums_from_words(a["int_sums"][r])
                sums[r] = (w[:4], int(a["band_count"][r]), w[4])
            else:
                f = [float(x) for x in a["float_sums"][r]]
                sums[r] = (f[:4], int(a["band_count"][r]), f[4])
            t, tb = fo.split_points(p, *sums[r])
            if p.exact:
                split[r], split_b[r] = t, tb
            else:
                centre[r], centre_b[r] = t, tb
        b = self.engine.first_order_splits_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, mode, base, split, split_b,
                                               centre, centre_b, band_lo, band_hi, stream=s.stream)
        out = []
        for r in rows:
            if r not in plan:
                out.append(fo.build_row(r, names[r], bw))
                continue
            p = plan[r]
            splits = [int(x) for x in b["below"][r]] if p.exact else [float(x) for x in b["abs_dev"][r]]
            ps, nb, sb = sums[r]
            out.append(fo.build_row(r, names[r], bw, p, a["histogram"][r][1:], ps, nb, sb, splits, s.spacing, shift))
        return fo.FirstOrderFeatures(s.spacing, bw, shift, out)

    def first_order_maps(self, image, mask, label="lung", features=None, kernel_radius=1, masked_kernel=True, bin_width=25,
                         voxel_array_shift=0, init_value=0.0, spacing=None):
        """PyRadiomics' voxel-based first-order extraction of one row -> lungmask_b200.first_order_maps.FirstOrderMaps:
        one float64 map of the volume's shape per feature of first_order.FIRST_ORDER_FEATURES (or of `features`, a
        subset, in that order), indexed by name (`fm["Entropy"]`).  `label`: a label value 1..255 or "lung" (mask > 0);
        the ROI is the row's voxels with a non-NaN value.  Each ROI voxel gets the features of the candidates of its
        window, the (2 kernel_radius + 1)^3 cube about it clipped at the array border (kernel_radius 1, 2 or 3): the
        window's ROI voxels (masked_kernel) or its non-NaN voxels.  Every other voxel holds `init_value`.  The levels of
        Entropy and Uniformity come from the fixed `bin_width` discretisation of the ROI (masked) or of the non-NaN voxels
        of its bounding box padded by kernel_radius (unmasked); more than 255 levels or a +-inf there is a ValueError
        before any map kernel runs.  The features and `voxel_array_shift`, `spacing` are those of `first_order`, formed
        per window in the sequence of DESIGN §4.15 (bit-identical to first_order_maps.maps_host).

        `image`, `mask` and `spacing` as for `first_order`.  CUDA inputs give CUDA float64 tensors on their device with no
        host copy, CPU tensors CPU tensors and everything else numpy arrays.  Each map takes 8 bytes per voxel (629 MB at
        300 x 512 x 512, 11.3 GB for all 18), allocated for the requested features only."""
        import torch
        from . import first_order as fo
        from . import first_order_maps as fm
        from . import texture as tx
        row = fm.check_label(label)
        feats = fm.check_features(features)
        r = fm.check_radius(kernel_radius)
        bw = tx.check_arguments(bin_width)
        shift = fo.check_shift(voxel_array_shift)
        s = self._stage("first_order_maps", image, mask, spacing)
        shape = tuple(s.mask.shape)
        code = 256 if row == fm.UNION else row
        integer = s.dtype in (_native.DTYPE_U8, _native.DTYPE_I8, _native.DTYPE_I16, _native.DTYPE_I32, _native.DTYPE_I64)
        n_roi, n_d, vmin, vmax, region, d_row = self._maps_region(s, code, r, masked_kernel, integer)
        plan = fm.plan_maps(n_d, vmin, vmax, bw, integer, shift, n_roi, "first_order_maps: row %s" % label)
        del region
        vv = float("nan") if s.spacing is None else (s.spacing[0] * s.spacing[1]) * s.spacing[2]
        K = (2 * r + 1) ** 3
        table = torch.from_numpy(fm.entropy_table(K)).to(s.mask.device)
        out = torch.empty((len(feats),) + shape, dtype=torch.float64, device=s.mask.device)
        # an empty ROI: the kernel writes init_value everywhere (no voxel reads the discretisation)
        self.engine.first_order_maps_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, code, r, masked_kernel, bw,
                                         plan.low or 0, plan.n_levels or 1, plan.exact, plan.base, shift, vv,
                                         float(init_value), fm.feature_bits(feats), table.data_ptr(), table.numel(),
                                         out.data_ptr(), stream=s.stream)
        maps = collections.OrderedDict((f, s.back(out[j])) for j, f in enumerate(feats))
        return fm.FirstOrderMaps(row, r, bool(masked_kernel), bw, shift, float(init_value), plan.low, plan.n_levels,
                                 plan.exact, n_roi, s.spacing, maps)

    def _maps_region(self, s, code, r, masked_kernel, integer):
        """The ROI count of row `code` (1..255, or 256 for mask > 0) of a staged feature-map call and its discretisation
        region D (DESIGN §4.15): the ROI (masked_kernel) or the non-NaN voxels of the ROI's bounding box padded by r.
        -> (n_roi, n_d, vmin, vmax, region, d_row): D is the voxels of the uint8 tensor `region` equal to d_row with a
        non-NaN value, n_d of them spanning [vmin, vmax]."""
        import torch
        shape = tuple(s.mask.shape)
        st = self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, s.mask.data_ptr(), shape, (), (), stream=s.stream)
        n_roi = int(st["voxels"][code] - st["nan_voxels"][code])
        d_row, region = code, s.mask
        if n_roi and not masked_kernel:   # D: the non-NaN voxels of the ROI's bounding box padded by r
            roi = s.mask > 0 if code == 256 else s.mask == code
            if not integer:
                roi &= ~torch.isnan(s.vol)
            box = []
            for ax in range(3):
                idx = torch.nonzero(roi.any(dim=[a for a in range(3) if a != ax])).reshape(-1)
                box.append(slice(max(int(idx[0]) - r, 0), int(idx[-1]) + r + 1))
            region = torch.zeros_like(s.mask)
            region[tuple(box)] = 1
            d_row = 1
            st = self.engine.label_stats_dev(s.vol.data_ptr(), s.dtype, region.data_ptr(), shape, (), (), stream=s.stream)
        n_d = int(st["voxels"][d_row] - st["nan_voxels"][d_row])
        return n_roi, n_d, float(st["moments"][d_row][2]), float(st["moments"][d_row][3]), region, d_row

    def glcm_maps(self, image, mask, label="lung", features=None, kernel_radius=1, masked_kernel=True, bin_width=25,
                  init_value=0.0):
        """PyRadiomics' voxel-based GLCM extraction of one row -> lungmask_b200.glcm_maps.GLCMMaps: one float64 map of
        the volume's shape per feature of texture.GLCM_FEATURES (or of `features`, a subset, in that order), indexed by
        name (`gm["Contrast"]`).  `label`, `kernel_radius` (1, 2 or 3), `masked_kernel` and the window are those of
        `first_order_maps`.  The discretisation region D (the ROI, or the non-NaN voxels of its bounding box padded by
        kernel_radius) is discretised with the fixed `bin_width` as `texture` does; more than 255 levels or a +-inf there
        is a ValueError before any map kernel runs.  For each of the 13 directions, a window's pairs are the voxel pairs
        (v, v + d) with both voxels among its candidates; the features of each direction with pairs follow the sequence
        of DESIGN §4.16 and are averaged over those directions (bit-identical to glcm_maps.maps_host).  An ROI voxel
        whose window has no pair gets NaN, every other voxel `init_value`.

        `image` and `mask` as for `texture` (a wavelet band or filtered image works as input).  CUDA inputs give CUDA
        float64 tensors on their device with no host copy, CPU tensors CPU tensors and everything else numpy arrays.  Each
        map takes 8 bytes per voxel (629 MB at 300 x 512 x 512, 13.8 GB for all 22), allocated for the requested features
        only."""
        import torch
        from . import first_order_maps as fm
        from . import glcm_maps as gm
        from . import texture as tx
        row = fm.check_label(label)
        feats = gm.check_features(features)
        r = fm.check_radius(kernel_radius)
        bw = tx.check_arguments(bin_width)
        s = self._stage("glcm_maps", image, mask)
        shape = tuple(s.mask.shape)
        code = 256 if row == fm.UNION else row
        integer = s.dtype in (_native.DTYPE_U8, _native.DTYPE_I8, _native.DTYPE_I16, _native.DTYPE_I32, _native.DTYPE_I64)
        n_roi, n_d, vmin, vmax, region, d_row = self._maps_region(s, code, r, masked_kernel, integer)
        low, ng = None, 0
        levels = torch.zeros(shape, dtype=torch.uint8, device=s.mask.device)
        if n_roi:
            low, ng = tx.discretisation(vmin, vmax, bw, "glcm_maps: row %s" % label)
            self.engine.texture_levels_dev(s.vol.data_ptr(), s.dtype, region.data_ptr(), shape, d_row, low, bw, ng,
                                           levels.data_ptr(), stream=s.stream)
        del region
        table = torch.from_numpy(fm.entropy_table(gm.max_pairs_n(r))).to(s.mask.device)
        out = torch.empty((len(feats),) + shape, dtype=torch.float64, device=s.mask.device)
        # an empty ROI: the level map is all 0, so every voxel gets init_value
        self.engine.glcm_maps_dev(levels.data_ptr(), s.mask.data_ptr(), shape, code, r, ng or 1, float(init_value),
                                  gm.feature_bits(feats), table.data_ptr(), table.numel(), out.data_ptr(), stream=s.stream)
        maps = collections.OrderedDict((f, s.back(out[j])) for j, f in enumerate(feats))
        return gm.GLCMMaps(row, r, bool(masked_kernel), bw, float(init_value), low, ng, n_roi, maps)

    def texture_maps(self, image, mask, classes=("glszm", "glrlm", "gldm", "ngtdm"), label="lung", features=None,
                     kernel_radius=1, masked_kernel=True, bin_width=25, gldm_alpha=0, init_value=0.0):
        """PyRadiomics' voxel-based GLSZM, GLRLM, GLDM and NGTDM extraction of one row ->
        lungmask_b200.texture_maps.TextureMaps: one float64 map of the volume's shape per feature of the `classes`,
        keyed by class-qualified PyRadiomics names (`tm["glszm_SmallAreaEmphasis"]`, `tm["ngtdm_Contrast"]`), or of
        `features`, a subset of those names, in class then feature order.  `classes` as for `texture`, without "glcm"
        (glcm_maps gives those).  `label`, `kernel_radius` (1, 2 or 3), `masked_kernel`, the window, the discretisation
        with the fixed `bin_width` and its refusals are those of `glcm_maps`.  Only voxels that are candidates of the window
        link: zones (26-connected, equal level), runs along the 13 directions (features averaged over them), dependence
        (neighbours within `gldm_alpha` levels, a non-negative int) and the NGTDM neighbourhoods.  Centres get their
        window's features in the sequence of DESIGN §4.17 (bit-identical to texture_maps.maps_host); NGTDM gives NaN where
        no candidate of the window has a neighbour.  Every other voxel holds `init_value`.

        `image` and `mask` as for `texture` (a wavelet band or filtered image works as input).  CUDA inputs give CUDA
        float64 tensors on their device with no host copy, CPU tensors CPU tensors and everything else numpy arrays.  The
        level map is built once per call.  Each map takes 8 bytes per voxel (629 MB at 300 x 512 x 512, 32 GB for all 51),
        allocated for the requested features only."""
        import torch
        from . import first_order_maps as fm
        from . import texture as tx
        from . import texture_maps as tm
        row = fm.check_label(label)
        cls = tm.check_classes(classes)
        feats = tm.check_features(features, cls)
        r = fm.check_radius(kernel_radius)
        bw = tx.check_arguments(bin_width)
        alpha = tx.check_alpha(gldm_alpha)
        s = self._stage("texture_maps", image, mask)
        shape = tuple(s.mask.shape)
        code = 256 if row == fm.UNION else row
        integer = s.dtype in (_native.DTYPE_U8, _native.DTYPE_I8, _native.DTYPE_I16, _native.DTYPE_I32, _native.DTYPE_I64)
        n_roi, n_d, vmin, vmax, region, d_row = self._maps_region(s, code, r, masked_kernel, integer)
        low, ng = None, 0
        levels = torch.zeros(shape, dtype=torch.uint8, device=s.mask.device)
        if n_roi:
            low, ng = tx.discretisation(vmin, vmax, bw, "texture_maps: row %s" % label)
            self.engine.texture_levels_dev(s.vol.data_ptr(), s.dtype, region.data_ptr(), shape, d_row, low, bw, ng,
                                           levels.data_ptr(), stream=s.stream)
        del region
        table = torch.from_numpy(fm.entropy_table((2 * r + 1) ** 3)).to(s.mask.device)
        out = torch.empty((len(feats),) + shape, dtype=torch.float64, device=s.mask.device)
        # one launch per class into its planes; an empty ROI: the level map is all 0, so every voxel gets init_value
        j = 0
        for c in cls:
            bits = tm.feature_bits(feats, c)
            if not bits:
                continue
            self.engine.texture_maps_dev(levels.data_ptr(), s.mask.data_ptr(), shape, code, r, ng or 1, tm.CLASS_CODES[c],
                                         alpha, float(init_value), bits, table.data_ptr(), table.numel(),
                                         out[j].data_ptr(), stream=s.stream)
            j += bin(bits).count("1")
        maps = collections.OrderedDict((f, s.back(out[k])) for k, f in enumerate(feats))
        return tm.TextureMaps(row, r, bool(masked_kernel), bw, float(init_value), low, ng, n_roi, cls, alpha, maps)

    def shape(self, mask, spacing=None, image=None):
        """Mesh shape features of every row of `statistics` -> lungmask_b200.shape.ShapeFeatures: every label value in the
        mask and every label 1..K-1 of the model (absent ones with 0 voxels and NaN features), then "lung" (mask != 0).
        A voxel is in label l's row when mask == l, so the fissures between lobes are surfaces of each lobe but interior
        to "lung".

        Each row is meshed by marching cubes on the mask padded with one voxel of outside, as PyRadiomics does: a lung cut
        by the first or last slice is closed there by a flat face (the opposite of `surface_distance`, where voxels
        outside the array are not background).  The 14 features of shape.SHAPE_FEATURES use PyRadiomics' names:
        SurfaceArea and MeshVolume of the mesh, VoxelVolume, SurfaceVolumeRatio, Sphericity, the maximum 3-D diameter and
        the maximum 2-D diameters within slices (equal axis-0 index), columns (axis 1) and rows (axis 2) between mesh
        vertices, and the principal axis lengths, Elongation and Flatness of the voxel positions.  Each row also holds
        the exact sums they come from (cube_counts, cube_possum, moments) and the squared diameters d2.

        `spacing` (x, y, z) in mm is required: given, or supplied by `image` (a Volume or SimpleITK image, used for
        nothing else); without one this is a ValueError before any kernel runs.  `mask`: (S, H, W) uint8 or bool, numpy,
        a CPU tensor, or a CUDA tensor on the engine's device read in place after the work queued on the current stream;
        it is left unchanged."""
        from . import shape as sh
        from .statistics import label_name
        if spacing is None and image is not None:
            spacing = tuple(image.spacing) if hasattr(image, "spacing") else tuple(image.GetSpacing())
        spacing = sh.check_spacing(spacing)
        s = self._stage("shape", None, mask, mask_only=True)
        shape = tuple(s.mask.shape)
        res = self.engine.shape_sums_dev(s.mask.data_ptr(), shape, stream=s.stream)
        present = set(int(x) for x in np.nonzero(res["moments"][1:256, 0])[0] + 1)
        rows = sorted(present | set(range(1, self.engine.n_classes[0]))) + [256]
        geometry = sh.config_geometry(spacing)
        out = []
        for r in rows:
            d2 = np.zeros(4)
            if r == 256 and present or r in present:
                d2 = self.engine.max_diameters_dev(s.mask.data_ptr(), shape, r, spacing[::-1], stream=s.stream)
            name = sh.UNION if r == 256 else label_name(self.modelname, r)
            out.append(sh.build_row(r, name, spacing, res["cube_counts"][r], res["cube_possum"][r], res["moments"][r], d2,
                                    geometry))
        return sh.ShapeFeatures(spacing, out)

    def mesh(self, mask, spacing=None, image=None, rows=None, space="lps"):
        """The marching-cubes surface of every row of `shape` -> lungmask_b200.mesh.MeshSet: every label value in the mask
        and every label 1..K-1 of the model (absent ones as empty meshes), then "lung" (mask != 0); or the rows named by
        `rows` (label values and / or "lung"), in that order.  Each is the mesh whose area and volume `shape` reports
        (DESIGN §4.14): vertices at cube-edge midpoints of the mask padded with one voxel of outside, triangles from
        shape.triangle_table(), closed and with normals pointing out of the row; not smoothed or decimated.

        Each Mesh holds `vertices` (float64 (V, 3), mm), `index2` (int32 (V, 3), the exact doubled array-axis coordinates)
        and `triangles` (int32 (T, 3)).  The positions are placed with the origin, direction and spacing of `image` (a
        Volume or SimpleITK image; `spacing` overrides its spacing), or with `spacing` (x, y, z) alone (origin 0, identity
        direction).  `space` "lps" (the frame of Volume and SimpleITK) or "ras" (the first two components negated).
        `mask`: (S, H, W) uint8 or bool, numpy or a CPU tensor (numpy arrays back), or a CUDA tensor on the engine's device
        read in place after the work queued on the current stream (tensors on that device back, with no host copy).  Bad
        spacing, rows, space or direction raise a ValueError before any kernel runs."""
        import torch
        from . import mesh as me
        from .statistics import label_name
        spacing, origin, direction = me.geometry(spacing, image)
        space = me.check_space(space)
        want = None if rows is None else me.check_rows(rows)
        s = self._stage("mesh", None, mask, mask_only=True)
        on_device = _is_tensor(mask) and mask.is_cuda
        shape, dev = tuple(s.mask.shape), s.mask.device
        present = self._mask_labels(s.mask, s.stream)
        order = want if want is not None else sorted(present | set(range(1, self.engine.n_classes[0]))) + [256]
        geo = me.geometry_vector(spacing, origin, direction)
        out = []
        for r in order:
            label = me.UNION if r == 256 else r
            nv = nt = 0
            if r in present or r == 256 and present:
                nv, nt = self.engine.mesh_counts_dev(s.mask.data_ptr(), shape, r, me.TABLE_OFFSETS, me.TABLE_CODES,
                                                     stream=s.stream)
                me.check_counts(label, nv, nt)
            index2 = torch.empty((nv, 3), dtype=torch.int32, device=dev)
            verts = torch.empty((nv, 3), dtype=torch.float64, device=dev)
            tris = torch.empty((nt, 3), dtype=torch.int32, device=dev)
            if nv or nt:
                self.engine.mesh_emit_dev(s.mask.data_ptr(), shape, r, me.TABLE_OFFSETS, me.TABLE_CODES, geo, nv, nt,
                                          index2.data_ptr(), verts.data_ptr(), tris.data_ptr(), ras=space == "ras",
                                          stream=s.stream)
            m = me.Mesh(label, me.UNION if r == 256 else label_name(self.modelname, r), verts, index2, tris, space)
            out.append(m if on_device else m.numpy())
        return me.MeshSet(spacing, origin, direction, space, out)

    def _mask_labels(self, mask, stream):
        """The non-zero label values of a (S,H,W) uint8 CUDA mask tensor.  lm_label_stats_dev with the mask as its own uint8
        volume and no percentiles or thresholds: its count and histogram passes over the mask bytes."""
        voxels = self.engine.label_stats_dev(mask.data_ptr(), _native.DTYPE_U8, mask.data_ptr(), mask.shape, (), (),
                                             stream=stream)["voxels"]
        return set(int(x) for x in np.nonzero(voxels[1:256])[0] + 1)

    def wavelet(self, image, wavelet="coif1", decompositions=None):
        """PyRadiomics' wavelet decompositions of `image` (getWaveletImage with its defaults: pywt.swtn, one level, start
        level 0) -> {name: float64 band of the image's shape}, in PyRadiomics' order: wavelet-LLH, -LHL, -LHH, -HLL,
        -HLH, -HHL, -HHH, then -LLL.  The letters are the filters along (x, y, z) = array axes (2, 1, 0) of the (S, H, W)
        array as given (no reorientation, as PyRadiomics filters sitk.GetArrayFromImage(image)).

        The values are converted to float64 and filtered along axis 2, then 1, then 0 by the periodic stationary
        transform: out[o] = sum_j f[j] in[(o + F/2 - j) mod N'], every product and sum rounded to float64, an odd axis
        wrapped to N' = N + 1 (index N holds index 0) and trimmed back; bit-identical to wavelet.swt_host.  `wavelet`:
        "coif1" (F = 6: every axis needs at least 5 voxels) or "haar" (F = 2).  `decompositions`: None for all 8, or a
        collection of names ("wavelet-LLL" or "LLL"); all 8 of a 300 x 512 x 512 volume take 5 GB.  A NaN or +-inf in
        the volume is a ValueError.

        `image`: a numpy array, a Volume or SimpleITK image (its array; numpy bands come back), a CPU tensor (CPU tensors
        come back), or a CUDA tensor on the engine's device, read in place after the work queued on the current stream
        (CUDA float64 tensors on that device come back).  The input is left unchanged."""
        import torch
        from . import wavelet as wv
        wavelet = wv.check_wavelet(wavelet)
        names = wv.check_decompositions(decompositions)
        s = self._stage("wavelet", image, None, image_only=True)
        shape = wv.check_shape(s.vol.shape, wavelet)
        in_place = _is_tensor(image) and image.is_cuda
        out = {}
        band = None
        for n in names:
            if band is None or in_place:   # host results are copied out of one device band; CUDA results are the bands
                band = torch.empty(shape, dtype=torch.float64, device=s.vol.device)
            self.engine.wavelet_dev(s.vol.data_ptr(), s.dtype, shape, wavelet, wv.band_code(n), band.data_ptr(),
                                    stream=s.stream)
            out[n] = s.back(band)
        return out

    def wavelet_features(self, image, mask, wavelet="coif1", bin_width=25,
                         classes=("firstorder", "glcm", "glszm", "glrlm", "gldm", "ngtdm"), gldm_alpha=0, spacing=None,
                         voxel_array_shift=0, distances=(1,), force2d=False, force2d_dimension=0, weighting_norm=None):
        """The first-order and texture features of every wavelet decomposition of `image` under `mask` ->
        lungmask_b200.wavelet.WaveletFeatures: for each of the 8 decompositions of `wavelet` (see `wavelet`), in
        PyRadiomics' order, the FirstOrderFeatures of `first_order` and the TextureFeatures of `texture` run on that
        band with the rows of `statistics`.  `vector(label)` gives a row's flat vector with PyRadiomics' keys such as
        wavelet-LLH_firstorder_Mean.

        `classes`: a non-empty collection of "firstorder", "glcm", "glszm", "glrlm", "gldm" and "ngtdm".  `bin_width`: a
        positive integer, or a dict giving one for every decomposition name ("wavelet-LLL" or "LLL"): wavelet-LLL scales
        values by about 2.8, so it may need a wider bin.  Every decomposition's rows are discretised before any
        first-order or texture kernel runs; a row with more than 255 levels is a ValueError naming the decomposition, the
        row and a sufficient bin width.  `gldm_alpha`, `voxel_array_shift`, `spacing`, and the neighbourhood settings
        `distances`, `force2d`, `force2d_dimension` and `weighting_norm`: as for `texture` and `first_order`.  Bad
        arguments raise before any kernel runs.

        `image`, `mask` and `spacing` as for `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the
        spacing), CPU tensors, or CUDA tensors on the engine's device read in place after the work queued on the current
        stream; both are left unchanged.  One float64 band of the volume's size is held on the device at a time."""
        import torch
        from . import first_order as fo
        from . import texture as tx
        from . import wavelet as wv
        wavelet = wv.check_wavelet(wavelet)
        widths = wv.check_bin_widths(bin_width)
        first, texture_classes = wv.check_classes(classes)
        alpha = tx.check_alpha(gldm_alpha)
        shift = fo.check_shift(voxel_array_shift)
        settings = tx.check_settings(distances, force2d, force2d_dimension, weighting_norm)
        s = self._stage("wavelet_features", image, mask, spacing)
        if texture_classes:
            tx.check_weighting_spacing(settings, s.spacing)
        shape = wv.check_shape(s.vol.shape, wavelet)
        band = torch.empty(shape, dtype=torch.float64, device=s.mask.device)

        def compute(name):
            self.engine.wavelet_dev(s.vol.data_ptr(), s.dtype, shape, wavelet, wv.band_code(name), band.data_ptr(),
                                    stream=s.stream)

        out = self._image_features("wavelet_features", s, band, wv.NAMES, compute, widths, first, texture_classes, shift,
                                   alpha, settings)
        computed = (("firstorder",) if first else ()) + texture_classes
        return wv.WaveletFeatures(wavelet, computed, s.spacing, shift, alpha, out)

    def _image_features(self, what, s, image, names, compute, widths, first, texture_classes, shift, alpha, settings):
        """The feature loop of wavelet_features and filtered_features over the derived images `names`: compute(name)
        writes image `name` to the float64 device tensor `image` of the staged volume's shape.  Every image's rows
        (those of `statistics`) are discretised first with §4.9's rule, so that a row with more than 255 levels is a
        ValueError naming the image, the row and a sufficient bin width before any first-order or texture kernel runs;
        then each image is recomputed and `first_order` (when `first`) and `texture` (on `texture_classes`, with the
        texture.Settings `settings`) run on it with the staged mask.  -> [wavelet.ImageFeatures] in the order of
        `names`."""
        from . import texture as tx
        from . import wavelet as wv
        from .statistics import label_name
        shape = tuple(image.shape)
        for name in names:   # every image's discretisation first: a refusal stops the call before any feature kernel
            compute(name)
            st = self.engine.label_stats_dev(image.data_ptr(), _native.DTYPE_F64, s.mask.data_ptr(), shape, (), (),
                                             stream=s.stream)
            present = set(int(x) for x in np.nonzero(st["voxels"][1:256])[0] + 1)
            for r in sorted(present | set(range(1, self.engine.n_classes[0]))) + [256]:
                if st["voxels"][r] - st["nan_voxels"][r]:
                    row = "%s row %s" % (name, "lung" if r == 256 else "%d (%s)" % (r, label_name(self.modelname, r)))
                    try:
                        tx.discretisation(float(st["moments"][r][2]), float(st["moments"][r][3]), widths[name], row)
                    except ValueError as ex:
                        raise ValueError(what + ": " + str(ex).split(": ", 1)[1]) from None
        out = []
        for name in names:
            compute(name)
            d = wv.ImageFeatures(name, widths[name])
            if first:
                d.first_order = self.first_order(image, s.mask, widths[name], s.spacing, shift)
            if texture_classes:
                d.texture = self.texture(image, s.mask, widths[name], s.spacing, texture_classes, alpha, settings.distances,
                                         settings.force2d_dimension is not None, settings.force2d_dimension or 0,
                                         settings.weighting_norm)
            out.append(d)
        return out

    def _filter_plan(self, s, names, spacing, use_spacing):
        """Checks the image types `names` against the staged volume before any image is written -> compute(name, out):
        writes image type `name` of the volume to the float64 device tensor `out`.  The range pass runs once (a NaN or
        +-inf is a ValueError), an all-zero volume is refused for square, logarithm and exponential, and the gradient
        needs its spacing.  Integer volumes within lungmask_b200.filters.table_span get each elementwise type as a
        device table of the numpy statement, built on first use."""
        import torch
        from . import filters as flt
        shape = flt.check_shape(s.vol.shape)
        grad_spacing = flt.gradient_spacing(spacing, use_spacing) if "gradient" in names else None
        elementwise = [n for n in names if n != "gradient"]
        lo = hi = 0.0
        if elementwise:
            lo, hi = self.engine.image_range_dev(s.vol.data_ptr(), s.dtype, shape, stream=s.stream)
            for n in elementwise:
                flt.check_range(n, lo, hi)
        span = flt.table_span(s.dtype, lo, hi) if elementwise else None
        tables = {}

        def compute(name, out):
            if name == "gradient":
                self.engine.gradient_dev(s.vol.data_ptr(), s.dtype, shape, grad_spacing, out.data_ptr(), stream=s.stream)
                return
            if span is None:
                self.engine.image_filter_dev(s.vol.data_ptr(), s.dtype, shape, name, flt.scalar(name, max(abs(lo), abs(hi))),
                                             out.data_ptr(), stream=s.stream)
                return
            if name not in tables:   # uploaded on the current stream, the one the call runs on
                tables[name] = torch.from_numpy(flt.table(name, *span)).to(out.device)
            self.engine.image_filter_dev(s.vol.data_ptr(), s.dtype, shape, name, 0.0, out.data_ptr(),
                                         table=(tables[name].data_ptr(), span[0], span[1]), stream=s.stream)

        return compute

    def filtered(self, image, image_types=None, spacing=None, gradient_use_spacing=True):
        """PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient image types of `image` (get<Type>Image
        with its defaults) -> {name: float64 image of the image's shape}, in that order: "square", "squareroot",
        "logarithm", "exponential", "gradient".  The (S, H, W) array is taken as given (no reorientation), converted to
        float64, with m = max|x| over the whole volume; lungmask_b200.filters.filter_host is the numpy statement.
        Integer volumes whose max - min is below 2^20 are bit-identical to it (a table of the statement); float and
        wider integer volumes are bit-identical for square, squareroot and gradient, and within DESIGN §4.13's ulp bound
        for logarithm and exponential (CUDA's log and exp).  `image_types`: None for all 5, or a collection of names.
        The gradient uses `spacing` (x, y, z) mm, or a Volume's or SimpleITK image's, unless gradient_use_spacing is
        False (spacing 1).  A NaN or +-inf in the volume, or an all-zero volume for square, logarithm or exponential, is
        a ValueError before any image is written.

        `image`: a numpy array, a Volume or SimpleITK image (numpy images come back), a CPU tensor (CPU tensors come
        back), or a CUDA tensor on the engine's device, read in place after the work queued on the current stream (CUDA
        float64 tensors on that device come back).  The input is left unchanged."""
        import torch
        from . import filters as flt
        names = flt.check_image_types(image_types)
        if spacing is None and not isinstance(image, np.ndarray) and not _is_tensor(image):
            spacing = tuple(image.spacing) if hasattr(image, "spacing") else tuple(image.GetSpacing())
        s = self._stage("filtered", image, None, image_only=True)
        compute = self._filter_plan(s, names, spacing, gradient_use_spacing)
        in_place = _is_tensor(image) and image.is_cuda
        out = {}
        buf = None
        for n in names:
            if buf is None or in_place:   # host results are copied out of one device image; CUDA results are the images
                buf = torch.empty(tuple(s.vol.shape), dtype=torch.float64, device=s.vol.device)
            compute(n, buf)
            out[n] = s.back(buf)
        return out

    def filtered_features(self, image, mask, image_types=None, bin_width=25,
                          classes=("firstorder", "glcm", "glszm", "glrlm", "gldm", "ngtdm"), gldm_alpha=0, spacing=None,
                          voxel_array_shift=0, gradient_use_spacing=True, distances=(1,), force2d=False, force2d_dimension=0,
                          weighting_norm=None):
        """The first-order and texture features of PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient
        image types of `image` under `mask` -> lungmask_b200.filters.FilteredFeatures: for each image type of
        `image_types` (None for all 5; see `filtered`), in PyRadiomics' order, the FirstOrderFeatures of `first_order`
        and the TextureFeatures of `texture` run on that image with the rows of `statistics`.  `vector(label)` gives a
        row's flat vector with PyRadiomics' keys such as square_firstorder_Mean or gradient_glcm_Contrast.

        `classes`: a non-empty collection of "firstorder", "glcm", "glszm", "glrlm", "gldm" and "ngtdm".  `bin_width`: a
        positive integer, or a dict giving one for every requested image type.  Every image's rows are discretised
        before any first-order or texture kernel runs; a row with more than 255 levels is a ValueError naming the image
        type, the row and a sufficient bin width.  `gldm_alpha`, `voxel_array_shift`, `spacing`, and the neighbourhood
        settings `distances`, `force2d`, `force2d_dimension` and `weighting_norm`: as for `texture` and `first_order`;
        the spacing is also the gradient's (see `filtered`).  Bad arguments raise before any kernel runs.

        `image`, `mask` and `spacing` as for `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the
        spacing), CPU tensors, or CUDA tensors on the engine's device read in place after the work queued on the current
        stream; both are left unchanged.  One float64 image of the volume's size is held on the device at a time."""
        import torch
        from . import filters as flt
        from . import first_order as fo
        from . import texture as tx
        names = flt.check_image_types(image_types)
        widths = flt.check_bin_widths(bin_width, names)
        first, texture_classes = flt.check_classes(classes)
        alpha = tx.check_alpha(gldm_alpha)
        shift = fo.check_shift(voxel_array_shift)
        settings = tx.check_settings(distances, force2d, force2d_dimension, weighting_norm)
        s = self._stage("filtered_features", image, mask, spacing)
        if texture_classes:
            tx.check_weighting_spacing(settings, s.spacing)
        compute = self._filter_plan(s, names, s.spacing, gradient_use_spacing)
        image_buf = torch.empty(tuple(s.vol.shape), dtype=torch.float64, device=s.mask.device)
        out = self._image_features("filtered_features", s, image_buf, names, lambda n: compute(n, image_buf), widths,
                                   first, texture_classes, shift, alpha, settings)
        computed = (("firstorder",) if first else ()) + texture_classes
        return flt.FilteredFeatures(computed, s.spacing, shift, alpha, bool(gradient_use_spacing), out)

    def _log_plan(self, s, sigmas, spacing):
        """Checks the sigmas, the spacing and the staged volume's shape before any image is written -> (compute(sigma,
        out): writes the LoG image of `sigma` to the float64 device tensor `out`, the two float64 work volumes it uses)."""
        import torch
        from . import laplacian as lg
        sp = lg.check_spacing(spacing)
        shape = lg.check_shape(s.vol.shape, sp, sigmas)
        work = [torch.empty(shape, dtype=torch.float64, device=s.vol.device) for _ in range(2)]

        def compute(sigma, out):
            self.engine.laplacian_of_gaussian_dev(s.vol.data_ptr(), s.dtype, shape, sp, sigma,
                                                  [w.data_ptr() for w in work], out.data_ptr(), stream=s.stream)

        return compute

    def log_images(self, image, sigma, spacing=None):
        """PyRadiomics' LoG image type of `image` (getLoGImage: ITK's LaplacianRecursiveGaussianImageFilter normalised
        across scale) -> {name: float64 image of the image's shape} in the order of `sigma`, named as PyRadiomics names
        them: log-sigma-1-0-mm-3D for sigma 1.  `sigma`: a size in mm or a non-empty collection of them.  The (S, H, W)
        array is taken as given (no reorientation), converted to float64, with `spacing` (x, y, z) mm or a Volume's or
        SimpleITK image's; lungmask_b200.laplacian.log_host is the numpy statement, and the result equals it bit for bit
        (DESIGN §4.20).  A sigma that is not finite and > 0, a repeated sigma, a missing spacing, an axis under 4 voxels
        or under ceil(sigma / spacing) + 1 voxels and 2^32 voxels or more are a ValueError before any image is written;
        a NaN or +-inf in the volume is a ValueError.

        `image`: a numpy array, a Volume or SimpleITK image (numpy images come back), a CPU tensor (CPU tensors come
        back), or a CUDA tensor on the engine's device, read in place after the work queued on the current stream (CUDA
        float64 tensors on that device come back).  The input is left unchanged.  The call holds two float64 work
        volumes of the image's size on the device."""
        import torch
        from . import laplacian as lg
        sigmas = lg.check_sigmas(sigma)
        if spacing is None and not isinstance(image, np.ndarray) and not _is_tensor(image):
            spacing = tuple(image.spacing) if hasattr(image, "spacing") else tuple(image.GetSpacing())
        lg.check_spacing(spacing)
        s = self._stage("log_images", image, None, image_only=True)
        compute = self._log_plan(s, sigmas, spacing)
        in_place = _is_tensor(image) and image.is_cuda
        out = {}
        buf = None
        for sg in sigmas:
            if buf is None or in_place:   # host results are copied out of one device image; CUDA results are the images
                buf = torch.empty(tuple(s.vol.shape), dtype=torch.float64, device=s.vol.device)
            compute(sg, buf)
            out[lg.image_name(sg)] = s.back(buf)
        return out

    def log_features(self, image, mask, sigma, bin_width=25,
                     classes=("firstorder", "glcm", "glszm", "glrlm", "gldm", "ngtdm"), gldm_alpha=0, spacing=None,
                     voxel_array_shift=0, distances=(1,), force2d=False, force2d_dimension=0, weighting_norm=None):
        """The first-order and texture features of PyRadiomics' LoG image type of `image` under `mask` ->
        lungmask_b200.laplacian.LogFeatures: for each sigma of `sigma` (mm; see `log_images`), in that order, the
        FirstOrderFeatures of `first_order` and the TextureFeatures of `texture` run on that image with the rows of
        `statistics`.  `vector(label)` gives a row's flat vector with PyRadiomics' keys such as
        log-sigma-1-0-mm-3D_firstorder_Mean.

        `classes`: a non-empty collection of "firstorder", "glcm", "glszm", "glrlm", "gldm" and "ngtdm".  `bin_width`: a
        positive integer, or a dict keyed by image name or sigma giving one for every sigma.  Every image's rows are
        discretised before any first-order or texture kernel runs; a row with more than 255 levels is a ValueError
        naming the image, the row and a sufficient bin width.  `gldm_alpha`, `voxel_array_shift`, `spacing`, and the
        neighbourhood settings `distances`, `force2d`, `force2d_dimension` and `weighting_norm`: as for `texture` and
        `first_order`; the spacing is also the filter's.  Bad arguments raise before any kernel runs.

        `image`, `mask` and `spacing` as for `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the
        spacing), CPU tensors, or CUDA tensors on the engine's device read in place after the work queued on the current
        stream; both are left unchanged.  One float64 image and two float64 work volumes of the volume's size are held
        on the device."""
        import torch
        from . import first_order as fo
        from . import laplacian as lg
        from . import texture as tx
        sigmas = lg.check_sigmas(sigma)
        widths = lg.check_bin_widths(bin_width, sigmas)
        first, texture_classes = lg.check_classes(classes)
        alpha = tx.check_alpha(gldm_alpha)
        shift = fo.check_shift(voxel_array_shift)
        settings = tx.check_settings(distances, force2d, force2d_dimension, weighting_norm)
        s = self._stage("log_features", image, mask, spacing)
        if texture_classes:
            tx.check_weighting_spacing(settings, s.spacing)
        compute = self._log_plan(s, sigmas, s.spacing)
        by_name = {lg.image_name(sg): sg for sg in sigmas}
        image_buf = torch.empty(tuple(s.vol.shape), dtype=torch.float64, device=s.mask.device)
        out = self._image_features("log_features", s, image_buf, list(by_name), lambda n: compute(by_name[n], image_buf),
                                   widths, first, texture_classes, shift, alpha, settings)
        computed = (("firstorder",) if first else ()) + texture_classes
        return lg.LogFeatures(sigmas, computed, s.spacing, shift, alpha, out)

    def resample(self, image, mask, resampled_spacing=(1, 1, 1), spacing=None, interpolator="bspline", pad_distance=5):
        """PyRadiomics' resampling of `image` and `mask` to `resampled_spacing` (x, y, z) mm (resampledPixelSpacing; an
        entry of 0 keeps that axis) with interpolator "bspline" (sitkBSpline, the default) or "nearest"
        (sitkNearestNeighbor) for the image and nearest neighbour for the mask -> lungmask_b200.resample.Resampled.  The
        grid covers the bounding box of mask > 0 padded by `pad_distance` output voxels, clamped to the image; when the
        spacing already equals the request (np.allclose) the pair is only cropped.  Points outside the input are 0.  The
        image keeps its dtype (integers clamped, then truncated toward zero) and the mask comes back as uint8;
        lungmask_b200.resample.resample_host is the numpy statement, and the result equals it bit for bit (DESIGN
        §4.19).  The result goes straight into the feature calls:
            r = inferer.resample(image, mask); inferer.texture(r.image, r.mask, spacing=r.spacing)

        `image` and `mask` as for `statistics`: numpy arrays, a Volume or SimpleITK image (which supplies the spacing
        unless `spacing` is given, and makes the result carry the new origin and the direction), CPU tensors, or CUDA
        tensors on the engine's device read in place after the work queued on the current stream; the image comes back
        in the same kind and neither input is modified.  The array is taken as given (no reorientation) and the mask
        must lie on the image's grid.  A NaN or +-inf in the image, an empty mask, a bad spacing or pad, mismatched
        shapes and 2^32 or more input or output voxels are a ValueError before any image is written.  The B-spline holds
        one float64 coefficient volume of the input's size on the device during the call."""
        import torch
        from . import resample as rsm
        rsm.check_interpolator(interpolator)
        pad = rsm.check_pad(pad_distance)
        requested = rsm.check_resampled_spacing(resampled_spacing)
        if _is_tensor(image):
            src_dtype = None
            is_bool = image.dtype == torch.bool
        else:   # a numpy array's or a Volume's dtype; a SimpleITK image is read as staged
            src_dtype = image.dtype if isinstance(image, np.ndarray) else getattr(getattr(image, "array", None), "dtype", None)
            is_bool = src_dtype == np.bool_
        if is_bool:
            raise TypeError("resample: a bool image has no interpolation; give the image as uint8 or pass it as the mask")
        s = self._stage("resample", image, mask, spacing)
        ms = rsm.check_spacing(s.spacing)
        shape = rsm.check_shape(s.vol.shape)
        counts = [self.engine.plane_label_counts_dev(s.mask.data_ptr(), shape, axis, stream=s.stream)[:, 256]
                  for axis in (2, 1, 0)]
        g = rsm.grid(shape, ms, requested, *rsm.bounding_box_of_counts(counts), pad)
        interp = "nearest" if g.crop else interpolator
        device = s.vol.device
        tables = [torch.from_numpy(t).to(device) for t in g.tables[::-1]]   # c_z, c_y, c_x
        coeff = None
        if interp == "bspline":
            coeff = torch.empty(shape, dtype=torch.float64, device=device)
            self.engine.bspline_coefficients_dev(s.vol.data_ptr(), s.dtype, shape, coeff.data_ptr(), stream=s.stream)
        elif s.vol.dtype.is_floating_point:
            self.engine.image_range_dev(s.vol.data_ptr(), s.dtype, shape, stream=s.stream)   # refuses a NaN or +-inf
        out = torch.empty(g.shape, dtype=s.vol.dtype, device=device)
        out_mask = torch.empty(g.shape, dtype=torch.uint8, device=device)
        self.engine.resample_dev(s.vol.data_ptr(), s.dtype, coeff.data_ptr() if coeff is not None else None,
                                 s.mask.data_ptr(), shape, [t.data_ptr() for t in tables], g.shape, interp, out.data_ptr(),
                                 out_mask.data_ptr(), stream=s.stream)
        del coeff
        img, m = out, out_mask
        if not (_is_tensor(image) and image.is_cuda):
            img, m = img.cpu(), m.cpu()
            if _is_tensor(image):
                if image.dtype == torch.bfloat16:   # staged as float32: the float32 value rounded once more
                    img = img.to(torch.bfloat16)
            else:
                img = img.numpy()
                if src_dtype in (np.uint16, np.uint32):   # staged as int32 / int64: the same values clamped once more
                    img = rsm.cast_host(img, src_dtype)
            if not _is_tensor(mask):
                m = m.numpy()
        origin = direction = None
        if not isinstance(image, np.ndarray) and not _is_tensor(image):
            origin = tuple(image.origin) if hasattr(image, "origin") else tuple(image.GetOrigin())
            direction = tuple(image.GetDirection())
            origin = rsm.new_origin(origin, direction, ms, g.start)
        return rsm.Resampled(img, m, g.spacing, g.start, origin, direction)

    def _stage(self, what, image, mask, spacing=None, mask_only=False, image_only=False):
        """The inputs of an analysis call as contiguous tensors on the engine's device -> _Staged.  CUDA tensors must be on
        the engine's device and are read in place; a CUDA volume needs a CUDA mask and the reverse.  Everything else is
        uploaded: numpy arrays, CPU tensors as their numpy arrays (bfloat16 widened to float32), a Volume or SimpleITK
        image, which also supplies the orientation and, unless `spacing` is given, the spacing.  The mask is uint8 or bool
        of the volume's shape.  mask_only: `image` is not used and the volume and its dtype code are None.  image_only:
        `mask` is not used, the mask is None and back(t) gives a result of the volume's shape in the type the volume came
        as.  Neither input is modified."""
        import torch
        if image_only:
            return self._stage_image(what, image)
        device = torch.device("cuda", self.engine.device)
        inputs = {"mask": mask} if mask_only else {"volume": image, "mask": mask}
        on_cuda = [_is_tensor(x) and x.is_cuda for x in inputs.values()]
        in_place = any(on_cuda)
        code, vol, dtype = "LPS", None, None
        if in_place:
            if not all(on_cuda):
                raise ValueError("%s: a CUDA tensor needs a CUDA tensor as partner (volume on %s, mask on %s)"
                                 % (what, getattr(image, "device", "host"), getattr(mask, "device", "host")))
            for name, x in inputs.items():
                if x.device.index != self.engine.device:
                    raise ValueError("%s: the %s tensor is on %s, the engine on cuda:%d" % (what, name, x.device, self.engine.device))
            m, back = mask.detach(), (lambda t: t)
            if not mask_only:
                vol = image.detach()
        else:
            m = np.asarray(mask.detach().numpy() if _is_tensor(mask) else mask)
            back = (lambda t: t.cpu()) if _is_tensor(mask) else (lambda t: t.cpu().numpy())
            if not mask_only:
                if _is_tensor(image):
                    image = image.detach()
                    image = (image.float() if image.dtype == torch.bfloat16 else image).numpy()
                vol = image
                if not isinstance(image, np.ndarray):
                    vol, code = self._array_and_orientation(image, what)
                    if spacing is None:
                        spacing = tuple(image.spacing) if hasattr(image, "spacing") else tuple(image.GetSpacing())
                vol = np.asarray(vol)
        if spacing is not None:
            spacing = tuple(float(s) for s in spacing)
            if len(spacing) != 3:
                raise ValueError("spacing must be (x, y, z), got %s" % (spacing,))
        if not mask_only and vol.ndim != 3:
            raise ValueError("%s: expected a (slices, H, W) volume, got shape %s" % (what, tuple(vol.shape)))
        if m.dtype not in ((torch.uint8, torch.bool) if _is_tensor(m) else (np.uint8, np.bool_)):
            raise TypeError("%s: the mask must be uint8 or bool, got %s" % (what, m.dtype))
        if mask_only and m.ndim != 3:
            raise ValueError("%s: expected a (slices, H, W) mask, got shape %s" % (what, tuple(m.shape)))
        if not mask_only and tuple(m.shape) != tuple(vol.shape):
            raise ValueError("%s: the mask's shape %s differs from the volume's %s" % (what, tuple(m.shape), tuple(vol.shape)))
        if in_place:
            if not mask_only:
                vol, dtype = vol.contiguous(), _tensor_dtype_code(vol)
            m = m.contiguous()
        else:
            if not mask_only:
                vol, dtype = _host_volume(vol, what)
            with warnings.catch_warnings():   # read-only arrays: the host tensors are only copied from
                warnings.simplefilter("ignore", UserWarning)
                vol = None if mask_only else torch.from_numpy(vol).to(device)
                m = torch.from_numpy(np.ascontiguousarray(m)).to(device)
        if m.dtype == torch.bool:
            m = m.view(torch.uint8)
        return _Staged(vol, dtype, m, torch.cuda.current_stream(device).cuda_stream, spacing, code, back)

    def _stage_image(self, what, image):
        """_stage's image_only mode: the volume alone, read in place as a CUDA tensor on the engine's device or uploaded
        (numpy arrays, CPU tensors as their numpy arrays with bfloat16 widened to float32, a Volume's or SimpleITK image's
        array as given, without reorientation).  The orientation is "LPS" and the spacing None."""
        import torch
        device = torch.device("cuda", self.engine.device)
        if _is_tensor(image) and image.is_cuda:
            if image.device.index != self.engine.device:
                raise ValueError("%s: the volume tensor is on %s, the engine on cuda:%d" % (what, image.device, self.engine.device))
            if image.dim() != 3:
                raise ValueError("%s: expected a (slices, H, W) volume, got shape %s" % (what, tuple(image.shape)))
            vol = image.detach().contiguous()
            dtype, back = _tensor_dtype_code(vol), (lambda t: t)
        else:
            if _is_tensor(image):
                image = image.detach()
                vol, back = (image.float() if image.dtype == torch.bfloat16 else image).numpy(), (lambda t: t.cpu())
            else:
                vol, back = self._array_and_orientation(image, what)[0], (lambda t: t.cpu().numpy())
            vol = np.asarray(vol)
            if vol.ndim != 3:
                raise ValueError("%s: expected a (slices, H, W) volume, got shape %s" % (what, tuple(vol.shape)))
            vol, dtype = _host_volume(vol, what)
            with warnings.catch_warnings():   # read-only arrays: the host tensor is only copied from
                warnings.simplefilter("ignore", UserWarning)
                vol = torch.from_numpy(vol).to(device)
        return _Staged(vol, dtype, None, torch.cuda.current_stream(device).cuda_stream, None, "LPS", back)


def apply(image, model=None, force_cpu=False, batch_size=20, volume_postprocessing=True, tqdm_disable=False):
    """Deprecated wrapper (lungmask/mask.py:235-255)."""
    warnings.warn("The function `apply` will be removed in a future version. Please use the LMInferer class!",
                  DeprecationWarning)
    inferer = LMInferer(force_cpu=force_cpu, batch_size=batch_size, volume_postprocessing=volume_postprocessing,
                        tqdm_disable=tqdm_disable)
    if model is not None:
        if not isinstance(model, NativeModel):
            model = NativeModel(model.state_dict())
        inferer.model = model
        inferer.engine.load_weights(0, model.blob, model.n_classes)
    return inferer.apply(image)


def apply_fused(image, basemodel="LTRCLobes", fillmodel="R231", force_cpu=False, batch_size=20,
                volume_postprocessing=True, tqdm_disable=False):
    """Deprecated wrapper (lungmask/mask.py:258-279)."""
    warnings.warn("The function `apply_fused` will be removed in a future version. Please use the LMInferer class!",
                  DeprecationWarning)
    inferer = LMInferer(modelname=basemodel, force_cpu=force_cpu, fillmodel=fillmodel, batch_size=batch_size,
                        volume_postprocessing=volume_postprocessing, tqdm_disable=tqdm_disable)
    return inferer.apply(image)
