"""Wavelet decompositions and their first-order and texture features per lung and lobe: the taps, names and argument
checks of LMInferer.wavelet and LMInferer.wavelet_features (lm_wavelet_dev; DESIGN §4.12), the numpy statement
swt_host, and the result WaveletFeatures.

The decomposition is PyRadiomics' getWaveletImage with its defaults: pywt.swtn, one level, start level 0, over the axes
(2, 1, 0) of the (S, H, W) array as given.  Every value is converted to float64; the x pass (array axis 2), the y pass
(axis 1) and the z pass (axis 0) each give out[o] = sum_{j=0..F-1} f[j] in[(o + F/2 - j) mod N'], summed from +0.0
with j ascending and every product and sum rounded to float64.  An odd axis of N voxels is wrapped to N' = N + 1 (index
N holds index 0) and the result is trimmed back to N.  The 8 decompositions are named and ordered as PyRadiomics yields
them; the letters are the filters along (x, y, z), so wavelet-LLH is high-pass along array axis 0.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

# PyWavelets' dec_lo; dec_hi[k] = (-1)^(k+1) dec_lo[F-1-k] (decomposition_filters).  The coif1 values are PyWavelets'
# table, which differs from the closed form by ~1e-12 relative.
DEC_LO = {
    "coif1": (-0.01565572813546454, -0.0727326195128539, 0.38486484686420286, 0.8525720202122554, 0.3378976624578092,
              -0.0727326195128539),
    "haar": (0.7071067811865476, 0.7071067811865476),
}
WAVELETS = tuple(DEC_LO)

NAMES = ("wavelet-LLH", "wavelet-LHL", "wavelet-LHH", "wavelet-HLL", "wavelet-HLH", "wavelet-HHL", "wavelet-HHH",
         "wavelet-LLL")


def band_code(name):
    """The band of lm_wavelet_dev of a decomposition name: 4 h_x + 2 h_y + h_z."""
    x, y, z = (1 if c == "H" else 0 for c in name[-3:])
    return 4 * x + 2 * y + z


FEATURE_CLASSES = ("firstorder", "glcm", "glszm", "glrlm", "gldm", "ngtdm")
MAX_VOXELS = 1 << 32


def decomposition_filters(wavelet):
    """-> (dec_lo, dec_hi) float64 arrays of a wavelet of WAVELETS."""
    lo = np.array(DEC_LO[check_wavelet(wavelet)], dtype=np.float64)
    F = lo.size
    hi = np.array([(1.0 if k % 2 else -1.0) * lo[F - 1 - k] for k in range(F)], dtype=np.float64)
    return lo, hi


def check_wavelet(wavelet):
    """-> the wavelet name; TypeError for a non-string, ValueError for a name not in WAVELETS."""
    if not isinstance(wavelet, str):
        raise TypeError("wavelet must be a name such as 'coif1', got %r" % (wavelet,))
    if wavelet not in DEC_LO:
        raise ValueError("wavelet: unknown wavelet %r (known: %s)" % (wavelet, ", ".join(WAVELETS)))
    return wavelet


def decomposition_name(name):
    """-> the full decomposition name of "LLH" or "wavelet-LLH"; ValueError for anything else."""
    if isinstance(name, str):
        full = name if name.startswith("wavelet-") else "wavelet-" + name
        if full in NAMES:
            return full
    raise ValueError("unknown wavelet decomposition %r (known: %s)" % (name, ", ".join(NAMES)))


def check_decompositions(decompositions):
    """-> the decomposition names in PyRadiomics' order: None means all 8, else a non-empty collection of names."""
    if decompositions is None:
        return NAMES
    if isinstance(decompositions, (str, bytes)):
        raise TypeError("decompositions must be a collection of names such as ('wavelet-LLL',), got the string %r"
                        % (decompositions,))
    names = [decomposition_name(d) for d in decompositions]
    if not names:
        raise ValueError("decompositions: at least one of %s is needed" % ", ".join(NAMES))
    return tuple(n for n in NAMES if n in names)


def check_shape(shape, wavelet):
    """ValueError for a volume that is not 3-D, has 2^32 voxels or more, or an axis whose padded extent is shorter than
    the filter (coif1: an axis of fewer than 5 voxels)."""
    shape = tuple(int(s) for s in shape)
    if len(shape) != 3:
        raise ValueError("wavelet: expected a (slices, H, W) volume, got shape %s" % (shape,))
    F = len(DEC_LO[check_wavelet(wavelet)])
    for a, n in enumerate(shape):
        if n + (n & 1) < F:
            raise ValueError("wavelet: axis %d of shape %s has %d voxels; %s needs a padded extent of at least %d"
                             % (a, shape, n, wavelet, F))
    if math.prod(shape) >= MAX_VOXELS:
        raise ValueError("wavelet: shape %s has 2^32 voxels or more" % (shape,))
    return shape


def check_bin_widths(bin_width):
    """-> {decomposition name: bin width} for all of NAMES: an int for every decomposition, or a dict giving one for
    every decomposition name ("wavelet-LLL" or "LLL")."""
    from .texture import check_arguments
    if not isinstance(bin_width, dict):
        bw = check_arguments(bin_width)
        return {n: bw for n in NAMES}
    out = {}
    for k, v in bin_width.items():
        name = decomposition_name(k)
        if name in out:
            raise ValueError("bin_width: decomposition %s given twice" % name)
        out[name] = check_arguments(v)
    missing = [n for n in NAMES if n not in out]
    if missing:
        raise ValueError("bin_width: no bin width for %s" % ", ".join(missing))
    return {n: out[n] for n in NAMES}


def parse_bin_widths(spec):
    """The bin widths of a command-line SPEC: "25" for every decomposition, or a default followed by per-decomposition
    overrides such as "25,LLL=50" -> the dict of check_bin_widths.  ValueError for a malformed SPEC."""
    default, widths = None, {}
    for part in (p.strip() for p in str(spec).split(",")):
        key, _, value = part.rpartition("=")
        try:
            bw = int(value)
        except ValueError:
            raise ValueError("bin width %r is not an integer" % (value,)) from None
        if key:
            widths[decomposition_name(key.strip())] = bw
        elif default is None and not widths:
            default = bw
        else:
            raise ValueError("%r: only the first entry may be a default bin width" % (spec,))
    if default is not None:
        widths = dict({n: default for n in NAMES}, **widths)
    return check_bin_widths(widths)


def check_classes(classes):
    """-> (first order wanted, texture classes tuple) of a non-empty collection of names of FEATURE_CLASSES."""
    from .texture import CLASSES
    if isinstance(classes, (str, bytes)):
        raise TypeError("classes must be a collection of names such as ('firstorder', 'glcm'), got the string %r"
                        % (classes,))
    names = list(classes)
    for c in names:
        if not isinstance(c, str):
            raise TypeError("classes: %r is not a name" % (c,))
        if c not in FEATURE_CLASSES:
            raise ValueError("classes: unknown feature class %r (known: %s)" % (c, ", ".join(FEATURE_CLASSES)))
    if not names:
        raise ValueError("classes: at least one of %s is needed" % ", ".join(FEATURE_CLASSES))
    return "firstorder" in names, tuple(c for c in CLASSES if c in names)


def ring_index(k, n):
    """The index an axis of n voxels is read at for the padded positions k: k mod N', and 0 for the pad index N of an
    odd axis (it holds index 0)."""
    m = np.asarray(k) % (n + (n & 1))
    return np.where(m == n, 0, m)


def swt_pass(a, taps, axis):
    """One periodic pass along `axis` of the float64 array `a`: out[o] = sum_j taps[j] a[(o + F/2 - j) mod N'], from
    +0.0 with j ascending, each product and sum rounded to float64."""
    F, n = len(taps), a.shape[axis]
    # ext[t] = a[(t - (F - 1 - F/2)) mod N']: tap j of output o reads ext[o + F - 1 - j]
    ext = np.take(a, ring_index(np.arange(n + F - 1) - (F - 1 - F // 2), n), axis=axis)
    out = np.zeros(a.shape, np.float64)
    sl = [slice(None)] * a.ndim
    for j in range(F):
        sl[axis] = slice(F - 1 - j, F - 1 - j + n)
        out = out + np.float64(taps[j]) * ext[tuple(sl)]
    return out


def swt_host(volume, wavelet="coif1", decompositions=None):
    """The numpy statement of LMInferer.wavelet: {name: float64 band} in PyRadiomics' order, the x and y passes shared
    between the bands that use them."""
    lo, hi = decomposition_filters(wavelet)
    names = check_decompositions(decompositions)
    v = np.asarray(volume)
    check_shape(v.shape, wavelet)
    v = v.astype(np.float64)
    out = {}
    for hx in (0, 1):
        want_x = [n for n in names if n[-3] == "LH"[hx]]
        if not want_x:
            continue
        X = swt_pass(v, (lo, hi)[hx], 2)
        for hy in (0, 1):
            want = [n for n in want_x if n[-2] == "LH"[hy]]
            if not want:
                continue
            Y = swt_pass(X, (lo, hi)[hy], 1)
            for n in want:
                out[n] = swt_pass(Y, (lo, hi)[n[-1] == "H"], 0)
    return {n: out[n] for n in names}


@dataclass
class ImageFeatures:
    """The features of one derived image: a wavelet decomposition here, an image type of lungmask_b200.filters."""
    name: str
    bin_width: int
    first_order: Optional[object] = None   # first_order.FirstOrderFeatures, None without "firstorder"
    texture: Optional[object] = None       # texture.TextureFeatures, None without a texture class

    def to_dict(self):
        return {"bin_width": self.bin_width,
                "firstorder": self.first_order.to_dict() if self.first_order is not None else None,
                "texture": self.texture.to_dict() if self.texture is not None else None}


WaveletDecomposition = ImageFeatures


def image_vector(images, classes, label):
    """The flat feature vector of a row over a list of ImageFeatures, with PyRadiomics' keys <image>_<class>_<feature>,
    in image, class (`classes`, in the order of FEATURE_CLASSES) and feature order."""
    from .first_order import FIRST_ORDER_FEATURES
    from .texture import GLCM_FEATURES, GLDM_FEATURES, GLRLM_FEATURES, GLSZM_FEATURES, NGTDM_FEATURES
    names = dict(zip(FEATURE_CLASSES, (FIRST_ORDER_FEATURES, GLCM_FEATURES, GLSZM_FEATURES, GLRLM_FEATURES,
                                       GLDM_FEATURES, NGTDM_FEATURES)))
    out = {}
    for d in images:
        for c in classes:
            f = d.first_order[label].features if c == "firstorder" else getattr(d.texture[label], c)
            for k in names[c]:
                out["%s_%s_%s" % (d.name, c, k)] = f[k]
    return out


@dataclass
class WaveletFeatures:
    wavelet: str
    classes: tuple                 # the computed classes, in the order of FEATURE_CLASSES
    spacing: Optional[tuple]
    voxel_array_shift: int
    gldm_alpha: int
    decompositions: list = field(default_factory=list)   # WaveletDecomposition per name of NAMES, in that order

    def __getitem__(self, name):
        """The WaveletDecomposition of "wavelet-LLH" (or "LLH")."""
        name = decomposition_name(name)
        for d in self.decompositions:
            if d.name == name:
                return d
        raise KeyError(name)

    @property
    def labels(self):
        """The row labels (those of `statistics`: each label, then "lung")."""
        d = self.decompositions[0]
        return [r.label for r in (d.first_order or d.texture).rows]

    def voxels(self, label):
        d = self.decompositions[0]
        return (d.first_order or d.texture)[label].voxels

    def vector(self, label):
        """The flat feature vector of a row with PyRadiomics' keys, such as wavelet-LLH_firstorder_Mean or
        wavelet-LLL_glcm_Contrast, in decomposition, class and feature order."""
        return image_vector(self.decompositions, self.classes, label)

    def to_dict(self):
        """JSON-ready: the to_dict() of every decomposition's FirstOrderFeatures and TextureFeatures (NaN as None)."""
        return {"wavelet": self.wavelet, "classes": list(self.classes),
                "spacing": list(self.spacing) if self.spacing is not None else None,
                "voxel_array_shift": self.voxel_array_shift, "gldm_alpha": self.gldm_alpha,
                "decompositions": {d.name: d.to_dict() for d in self.decompositions}}
