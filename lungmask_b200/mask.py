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

    def _mask_labels(self, mask, stream):
        """The non-zero label values of a (S,H,W) uint8 CUDA mask tensor.  lm_label_stats_dev with the mask as its own uint8
        volume and no percentiles or thresholds: its count and histogram passes over the mask bytes."""
        voxels = self.engine.label_stats_dev(mask.data_ptr(), _native.DTYPE_U8, mask.data_ptr(), mask.shape, (), (),
                                             stream=stream)["voxels"]
        return set(int(x) for x in np.nonzero(voxels[1:256])[0] + 1)

    def _stage(self, what, image, mask, spacing=None, mask_only=False):
        """The inputs of an analysis call as contiguous tensors on the engine's device -> _Staged.  CUDA tensors must be on
        the engine's device and are read in place; a CUDA volume needs a CUDA mask and the reverse.  Everything else is
        uploaded: numpy arrays, CPU tensors as their numpy arrays (bfloat16 widened to float32), a Volume or SimpleITK
        image, which also supplies the orientation and, unless `spacing` is given, the spacing.  The mask is uint8 or bool
        of the volume's shape.  mask_only: `image` is not used and the volume and its dtype code are None.  Neither input
        is modified."""
        import torch
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
