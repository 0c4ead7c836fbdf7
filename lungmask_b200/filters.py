"""PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient image types and their first-order and texture
features per lung and lobe: the names, argument checks, the numpy statement filter_host, the integer tables and the
result FilteredFeatures of LMInferer.filtered and LMInferer.filtered_features (lm_image_range_dev, lm_image_filter_dev,
lm_gradient_dev; DESIGN §4.13).

Each image type is PyRadiomics' get<Type>Image with its defaults on the (S, H, W) array as given, converted to float64,
with m = max|x| over the whole volume:
  square       c = 1 / sqrt(m); (c x)^2
  squareroot   c = m; x > 0: sqrt(x c), x < 0: -sqrt(-x c), anything else kept (-0.0 stays -0.0)
  logarithm    x > 0: log(x + 1), x < 0: -log(-(x - 1)), 0 kept; then y (m / max|y|)
  exponential  c = log(m) / m; exp(c x)
  gradient     ITK's GradientMagnitudeImageFilter with the image spacing: per axis (x = array axis 2, y = 1, z = 0)
               g = ((0 + k0 f[-1]) + k1 f[0]) + k2 f[+1], (k0, k1, k2) = (-0.5, 0, 0.5) (1 / s), neighbours outside the
               array clamped to the edge voxel; then sqrt(((0 + gx^2) + gy^2) + gz^2)
A NaN or +-inf anywhere in the volume is a ValueError, and so is m = 0 for square, logarithm and exponential (numpy gives
a NaN image there).
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from .wavelet import FEATURE_CLASSES, ImageFeatures, check_classes, image_vector  # noqa: F401  (re-exported)

NAMES = ("square", "squareroot", "logarithm", "exponential", "gradient")   # PyRadiomics' order and key prefixes
ELEMENTWISE = NAMES[:4]
NEEDS_NONZERO = ("square", "logarithm", "exponential")
MAX_VOXELS = 1 << 32
TABLE_SPAN = 1 << 20   # integer volumes with max - min below this go through a table of the numpy statement
# The most float64 ulps by which logarithm and exponential computed on the device (float and wider integer volumes:
# CUDA's log / exp, within 1 ulp, against numpy's, within 4) can differ from filter_host; derived in DESIGN §4.13.
ULP_BOUND = {"logarithm": 12, "exponential": 10}


def check_image_types(image_types):
    """-> the image type names in PyRadiomics' order: None means all 5, else a non-empty collection of NAMES."""
    if image_types is None:
        return NAMES
    if isinstance(image_types, (str, bytes)):
        raise TypeError("image_types must be a collection of names such as ('square', 'gradient'), got the string %r"
                        % (image_types,))
    names = list(image_types)
    for n in names:
        if n not in NAMES:
            raise ValueError("unknown image type %r (known: %s)" % (n, ", ".join(NAMES)))
    if not names:
        raise ValueError("image_types: at least one of %s is needed" % ", ".join(NAMES))
    return tuple(n for n in NAMES if n in names)


def check_bin_widths(bin_width, names=NAMES):
    """-> {image type: bin width} for `names`: an int for every image type, or a dict giving one for each of `names`
    (entries for other known image types are allowed and unused)."""
    from .texture import check_arguments
    if not isinstance(bin_width, dict):
        bw = check_arguments(bin_width)
        return {n: bw for n in names}
    out = {}
    for k, v in bin_width.items():
        if k not in NAMES:
            raise ValueError("bin_width: unknown image type %r (known: %s)" % (k, ", ".join(NAMES)))
        out[k] = check_arguments(v)
    missing = [n for n in names if n not in out]
    if missing:
        raise ValueError("bin_width: no bin width for %s" % ", ".join(missing))
    return {n: out[n] for n in names}


def parse_bin_widths(spec):
    """The bin widths of a command-line SPEC: "25" for every image type, or a default followed by per-type overrides
    such as "25,gradient=10" -> the dict of check_bin_widths.  ValueError for a malformed SPEC."""
    default, widths = None, {}
    for part in (p.strip() for p in str(spec).split(",")):
        key, _, value = part.rpartition("=")
        try:
            bw = int(value)
        except ValueError:
            raise ValueError("bin width %r is not an integer" % (value,)) from None
        key = key.strip()
        if key:
            if key not in NAMES:
                raise ValueError("unknown image type %r (known: %s)" % (key, ", ".join(NAMES)))
            widths[key] = bw
        elif default is None and not widths:
            default = bw
        else:
            raise ValueError("%r: only the first entry may be a default bin width" % (spec,))
    if default is not None:
        widths = dict({n: default for n in NAMES}, **widths)
    return check_bin_widths(widths, tuple(n for n in NAMES if n in widths))


def check_shape(shape):
    """ValueError for a volume that is not 3-D, is empty or has 2^32 voxels or more."""
    shape = tuple(int(s) for s in shape)
    if len(shape) != 3:
        raise ValueError("filters: expected a (slices, H, W) volume, got shape %s" % (shape,))
    if min(shape) < 1:
        raise ValueError("filters: shape %s is empty" % (shape,))
    if math.prod(shape) >= MAX_VOXELS:
        raise ValueError("filters: shape %s has 2^32 voxels or more" % (shape,))
    return shape


def gradient_spacing(spacing, use_spacing=True):
    """The (x, y, z) spacing of the gradient: (1, 1, 1) without use_spacing, else 3 finite positive sizes in mm;
    ValueError when it is missing or malformed."""
    if not use_spacing:
        return (1.0, 1.0, 1.0)
    if spacing is None:
        raise ValueError("gradient: the image spacing is needed (gradient_use_spacing=True); pass spacing=(x, y, z) in mm, "
                         "a Volume or SimpleITK image, or gradient_use_spacing=False")
    sp = tuple(float(s) for s in spacing)
    if len(sp) != 3 or not all(math.isfinite(s) and s > 0 for s in sp):
        raise ValueError("gradient: spacing must be 3 finite positive sizes (x, y, z) in mm, got %s" % (spacing,))
    return sp


def check_range(name, lo, hi):
    """ValueError when image type `name` is not defined for a volume of min `lo` and max `hi` (m = 0: numpy's statement
    gives NaN)."""
    if name in NEEDS_NONZERO and max(abs(lo), abs(hi)) == 0.0:
        raise ValueError("%s: the volume is all zeros (max |x| = 0), where %s is not defined" % (name, name))


def scalar(name, m):
    """The host scalar of an elementwise image type for m = max|x|, in numpy float64 as PyRadiomics forms it (the
    Logarithm scale m / max|y| is m / log(m + 1))."""
    m = np.float64(m)
    if name == "square":
        return float(1 / np.sqrt(m))
    if name == "squareroot":
        return float(m)
    if name == "logarithm":
        return float(m / np.log(m + 1))
    if name == "exponential":
        return float(np.log(m) / m)
    raise ValueError("unknown elementwise image type %r" % (name,))


def elementwise_host(v, name):
    """The numpy statement of an elementwise image type on the float64 array `v` (PyRadiomics' code, m over `v`)."""
    im = np.array(v, dtype=np.float64)
    m = np.max(np.abs(im))
    if name == "square":
        coeff = 1 / np.sqrt(m)
        return (coeff * im) ** 2
    if name == "squareroot":
        coeff = m
        im[im > 0] = np.sqrt(im[im > 0] * coeff)
        im[im < 0] = - np.sqrt(-im[im < 0] * coeff)
        return im
    if name == "logarithm":
        im[im > 0] = np.log(im[im > 0] + 1)
        im[im < 0] = - np.log(- (im[im < 0] - 1))
        return im * (m / np.max(np.abs(im)))
    if name == "exponential":
        coeff = np.log(m) / m
        return np.exp(coeff * im)
    raise ValueError("unknown elementwise image type %r" % (name,))


def gradient_host(v, spacing_xyz):
    """The numpy statement of the gradient magnitude of the float64 (S, H, W) array `v` with spacing (x, y, z)."""
    v = np.asarray(v, dtype=np.float64)
    a = np.zeros(v.shape, np.float64)
    for s, axis in zip(spacing_xyz, (2, 1, 0)):
        inv = np.float64(1.0) / np.float64(s)
        k0, k1, k2 = np.float64(-0.5) * inv, np.float64(0.0) * inv, np.float64(0.5) * inv
        i = np.arange(v.shape[axis])
        fm = np.take(v, np.maximum(i - 1, 0), axis=axis)
        fp = np.take(v, np.minimum(i + 1, v.shape[axis] - 1), axis=axis)
        g = ((np.float64(0.0) + k0 * fm) + k1 * v) + k2 * fp
        a = a + g * g
    return np.sqrt(a)


def filter_host(volume, type, spacing=None, use_spacing=True):
    """The numpy statement of LMInferer.filtered for one image type: the float64 image of `volume` (any real dtype, as
    float64).  `spacing` (x, y, z) mm is needed by "gradient" unless use_spacing is False.  ValueError for a NaN or +-inf,
    for m = 0 where the type is not defined, and for an unknown type."""
    if type not in NAMES:
        raise ValueError("unknown image type %r (known: %s)" % (type, ", ".join(NAMES)))
    v = np.asarray(volume)
    check_shape(v.shape)
    v = v.astype(np.float64)
    if not np.all(np.isfinite(v)):
        raise ValueError("%s: the volume holds a NaN or +-inf" % type)
    if type == "gradient":
        return gradient_host(v, gradient_spacing(spacing, use_spacing))
    check_range(type, float(v.min()), float(v.max()))
    return elementwise_host(v, type)


def table_span(dtype_code, lo, hi):
    """(first value, length) of the table of an integer volume of LM_DTYPE_* `dtype_code` with min `lo` and max `hi`,
    or None when it computes on the device instead: float dtypes, max - min >= 2^20, or |min|, |max| >= 2^53 (where
    the float64 min and max might not be the integers)."""
    from . import _native
    if dtype_code not in (_native.DTYPE_U8, _native.DTYPE_I8, _native.DTYPE_I16, _native.DTYPE_I32, _native.DTYPE_I64):
        return None
    if max(abs(lo), abs(hi)) >= 2.0 ** 53 or hi - lo >= TABLE_SPAN:
        return None
    return int(lo), int(hi) - int(lo) + 1


def table(name, first, length):
    """The numpy statement of an elementwise image type applied to first .. first + length - 1 as float64: the value of
    every voxel of an integer volume whose min and max are the ends (m and the scalars depend only on them)."""
    return elementwise_host(np.arange(first, first + length, dtype=np.int64).astype(np.float64), name)


@dataclass
class FilteredFeatures:
    classes: tuple                 # the computed classes, in the order of FEATURE_CLASSES
    spacing: Optional[tuple]
    voxel_array_shift: int
    gldm_alpha: int
    gradient_use_spacing: bool
    images: list = field(default_factory=list)   # wavelet.ImageFeatures per image type, in the order of NAMES

    def __getitem__(self, name):
        """The ImageFeatures of image type `name`."""
        for d in self.images:
            if d.name == name:
                return d
        raise KeyError(name)

    @property
    def labels(self):
        """The row labels (those of `statistics`: each label, then "lung")."""
        d = self.images[0]
        return [r.label for r in (d.first_order or d.texture).rows]

    def voxels(self, label):
        d = self.images[0]
        return (d.first_order or d.texture)[label].voxels

    def vector(self, label):
        """The flat feature vector of a row with PyRadiomics' keys, such as square_firstorder_Mean or
        gradient_glcm_Contrast, in image type, class and feature order."""
        return image_vector(self.images, self.classes, label)

    def to_dict(self):
        """JSON-ready: the to_dict() of every image type's FirstOrderFeatures and TextureFeatures (NaN as None)."""
        return {"classes": list(self.classes), "spacing": list(self.spacing) if self.spacing is not None else None,
                "voxel_array_shift": self.voxel_array_shift, "gldm_alpha": self.gldm_alpha,
                "gradient_use_spacing": self.gradient_use_spacing,
                "images": {d.name: d.to_dict() for d in self.images}}
