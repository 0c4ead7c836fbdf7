"""PyRadiomics' LoG image type (getLoGImage) and its first-order and texture features per lung and lobe: the names, the
argument checks, the recursive Gaussian coefficients, the numpy statement log_host and the result LogFeatures of
LMInferer.log_images and LMInferer.log_features (lm_laplacian_of_gaussian_dev; DESIGN §4.20).

For each sigma (mm) the image is ITK's LaplacianRecursiveGaussianImageFilter with NormalizeAcrossScale on and the image
spacing, on the (S, H, W) array as given (no reorientation), converted to float64.  Axes are in ITK order: d = x, y, z
are array axes 2, 1, 0 with spacing (x, y, z) in mm.

Coefficients (ITK's RecursiveGaussianImageFilter::SetUp, Deriche's 4th-order approximation), per axis in float64 with
sd = sigma / s_d, each operation rounded on its own in the order written:
  A1 = (1.3530, -0.6724, -1.3563)  B1 = (1.8151, -3.4327, 5.2318)  W1 = 0.6681  L1 = -1.3932
  A2 = (-0.3531, 0.6724, 0.3446)   B2 = (0.0902, 0.6100, -2.2355)  W2 = 2.0787  L2 = -1.3732
  N(a1, b1, a2, b2) with S_k = sin(W_k / sd), C_k = cos(W_k / sd), E_k = exp(L_k / sd):
    N0 = a1 + a2
    N1 = E2 (b2 S2 - (a2 + 2 a1) C2);  N1 += E1 (b1 S1 - (a1 + 2 a2) C1)
    N2 = (a1 + a2) C2 C1;  N2 -= b1 C2 S1 + b2 C1 S2;  N2 *= 2 E1 E2;  N2 += a2 E1 E1 + a1 E2 E2
    N3 = E2 E1 E1 (b2 S2 - a2 C2);  N3 += E1 E2 E2 (b1 S1 - a1 C1)
    SN = N0 + N1 + N2 + N3,  DN = N1 + 2 N2 + 3 N3,  EN = N1 + 4 N2 + 9 N3
  D1 = -2 E2 C2 - 2 E1 C1              D2 = 4 C2 C1 E1 E2 + E1 E1 + E2 E2
  D3 = -2 C1 E1 E2 E2 - 2 C2 E2 E1 E1  D4 = E1 E1 E2 E2
  SD = 1 + D1 + D2 + D3 + D4,  DD = D1 + 2 D2 + 3 D3 + 4 D4,  ED = D1 + 4 D2 + 9 D3 + 16 D4
  order 0 (smoothing): N of index 0; alpha0 = 2 SN / SD - N0; every N_i /= alpha0
  order 2 (the derivative axis): N' of index 0 and N'' of index 2;
    beta = -(2 SN'' - SD N0'') / (2 SN' - SD N0');  N_i = N''_i + beta N'_i, and SN, DN, EN likewise
    alpha2 = (EN SD SD - ED SN SD - 2 DN DD SD + 2 DD DD SN) / (SD SD SD);  every N_i *= sd sd / alpha2
  M1 = N1 - D1 N0, M2 = N2 - D2 N0, M3 = N3 - D3 N0, M4 = -D4 N0
  BN_i = D_i (N0 + N1 + N2 + N3) / SD,  BM_i = D_i (M1 + M2 + M3 + M4) / SD

Line filter (ITK's RecursiveSeparableImageFilter::FilterDataArray) of x[0 .. L-1], v = x[0], w = x[L-1], with
E(a1,b1, .., a4,b4) = ((a1 b1 + a2 b2) + a3 b3) + a4 b4:
  causal, taps before the line read v:
    y[0] = E(v,N0, v,N1, v,N2, v,N3) - E(v,BN1, v,BN2, v,BN3, v,BN4)
    y[1] = E(x[1],N0, v,N1, v,N2, v,N3) - E(y[0],D1, v,BN2, v,BN3, v,BN4)
    y[2] = E(x[2],N0, x[1],N1, v,N2, v,N3) - E(y[1],D1, y[0],D2, v,BN3, v,BN4)
    y[3] = E(x[3],N0, x[2],N1, x[1],N2, v,N3) - E(y[2],D1, y[1],D2, y[0],D3, v,BN4)
    y[i] = E(x[i],N0, x[i-1],N1, x[i-2],N2, x[i-3],N3) - E(y[i-1],D1, .., y[i-4],D4)        i = 4 .. L-1
  anticausal, on x again, taps after the line read w:
    z[L-1] = E(w,M1, w,M2, w,M3, w,M4) - E(w,BM1, w,BM2, w,BM3, w,BM4)
    z[L-2] = E(x[L-1],M1, w,M2, w,M3, w,M4) - E(z[L-1],D1, w,BM2, w,BM3, w,BM4)
    z[L-3] = E(x[L-2],M1, x[L-1],M2, w,M3, w,M4) - E(z[L-2],D1, z[L-1],D2, w,BM3, w,BM4)
    z[L-4] = E(x[L-3],M1, x[L-2],M2, x[L-1],M3, w,M4) - E(z[L-3],D1, z[L-2],D2, z[L-1],D3, w,BM4)
    z[i-1] = E(x[i],M1, x[i+1],M2, x[i+2],M3, x[i+3],M4) - E(z[i],D1, .., z[i+3],D4)      i = L-4 .. 1
  output y[i] + z[i]
Laplacian: for d = x, y, z: order 0 along the two other axes in x, y, z order, then order 2 along d; the terms are
added to a sum that starts at +0.0 in the order x, y, z.

Refused with a ValueError: a sigma that is not finite and > 0, an empty sigma list or two sigmas with one name, a
missing or non-positive spacing, an axis under 4 voxels, an axis d with size_d < ceil(sigma / s_d) + 1 (PyRadiomics
skips such a sigma with a warning), a NaN or +-inf in the volume and 2^32 voxels or more.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from .wavelet import FEATURE_CLASSES, ImageFeatures, check_classes, image_vector  # noqa: F401  (re-exported)

MAX_VOXELS = 1 << 32
MIN_EXTENT = 4
A1 = (1.3530, -0.6724, -1.3563)
B1 = (1.8151, -3.4327, 5.2318)
W1 = 0.6681
L1 = -1.3932
A2 = (-0.3531, 0.6724, 0.3446)
B2 = (0.0902, 0.6100, -2.2355)
W2 = 2.0787
L2 = -1.3732


def image_name(sigma):
    """PyRadiomics' image name of a sigma: 'log-sigma-%s-mm-3D' % str(float(sigma)).replace('.', '-')."""
    return "log-sigma-%s-mm-3D" % str(float(sigma)).replace(".", "-")


def check_sigmas(sigma):
    """-> the sigmas as floats in the given order: a non-empty collection (or one number) of finite sigmas > 0 mm with
    distinct image names."""
    if isinstance(sigma, (str, bytes)):
        raise TypeError("sigma must be a number or a collection of numbers in mm, got the string %r" % (sigma,))
    values = [sigma] if np.ndim(sigma) == 0 else list(np.asarray(sigma, dtype=object).ravel())
    if not values:
        raise ValueError("sigma: at least one sigma in mm is needed")
    out, names = [], set()
    for s in values:
        if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, float, np.integer, np.floating)):
            raise TypeError("sigma: %r is not a number" % (s,))
        f = float(s)
        if not (math.isfinite(f) and f > 0):
            raise ValueError("sigma: %r is not a finite size > 0 mm" % (s,))
        if image_name(f) in names:
            raise ValueError("sigma: %s is given twice (image %s)" % (f, image_name(f)))
        names.add(image_name(f))
        out.append(f)
    return tuple(out)


def check_spacing(spacing):
    """The (x, y, z) spacing in mm: 3 finite positive sizes; ValueError when it is missing or malformed."""
    if spacing is None:
        raise ValueError("log: the image spacing is needed; pass spacing=(x, y, z) in mm, a Volume or SimpleITK image")
    sp = tuple(float(s) for s in spacing)
    if len(sp) != 3 or not all(math.isfinite(s) and s > 0 for s in sp):
        raise ValueError("log: spacing must be 3 finite positive sizes (x, y, z) in mm, got %s" % (spacing,))
    return sp


def check_shape(shape, spacing=None, sigmas=()):
    """ValueError for a volume that is not 3-D, has an axis under 4 voxels or 2^32 voxels or more, and for a sigma whose
    ceil(sigma / s_d) + 1 exceeds the size of axis d (spacing (x, y, z))."""
    shape = tuple(int(s) for s in shape)
    if len(shape) != 3:
        raise ValueError("log: expected a (slices, H, W) volume, got shape %s" % (shape,))
    if min(shape) < MIN_EXTENT:
        raise ValueError("log: shape %s has an axis under %d voxels" % (shape, MIN_EXTENT))
    if math.prod(shape) >= MAX_VOXELS:
        raise ValueError("log: shape %s has 2^32 voxels or more" % (shape,))
    if spacing is not None:
        for sigma in sigmas:
            for d, (s, n) in enumerate(zip(spacing, shape[::-1])):
                need = math.ceil(sigma / s) + 1
                if n < need:
                    raise ValueError("log: sigma %s mm needs at least ceil(sigma / spacing) + 1 = %d voxels along %s "
                                     "(spacing %g mm), the volume has %d" % (sigma, need, "xyz"[d], s, n))
    return shape


def check_bin_widths(bin_width, sigmas):
    """-> {image name: bin width} for `sigmas`: an int for every image, or a dict keyed by image name or sigma giving
    one for each of them (entries for other sigmas are allowed and unused)."""
    from .texture import check_arguments
    names = [image_name(s) for s in sigmas]
    if not isinstance(bin_width, dict):
        bw = check_arguments(bin_width)
        return {n: bw for n in names}
    out = {}
    for k, v in bin_width.items():
        if isinstance(k, str) and k.startswith("log-sigma-"):
            key = k
        else:
            try:
                key = image_name(k)
            except (TypeError, ValueError):
                raise ValueError("bin_width: %r is neither a sigma nor a LoG image name" % (k,)) from None
        out[key] = check_arguments(v)
    missing = [n for n in names if n not in out]
    if missing:
        raise ValueError("bin_width: no bin width for %s" % ", ".join(missing))
    return {n: out[n] for n in names}


def parse_sigmas(spec):
    """The sigmas of a command-line SPEC such as "1,2,3,4,5" -> check_sigmas' tuple.  ValueError for a malformed SPEC."""
    values = []
    for part in (p.strip() for p in str(spec).split(",")):
        try:
            values.append(float(part))
        except ValueError:
            raise ValueError("sigma %r is not a number" % (part,)) from None
    return check_sigmas(values)


def parse_bin_widths(spec, sigmas):
    """The bin widths of a command-line SPEC for `sigmas`: "25" for every image, or a default followed by per-sigma
    overrides such as "25,3.0=50" -> the dict of check_bin_widths.  ValueError for a malformed SPEC."""
    default, widths = None, {}
    for part in (p.strip() for p in str(spec).split(",")):
        key, _, value = part.rpartition("=")
        try:
            bw = int(value)
        except ValueError:
            raise ValueError("bin width %r is not an integer" % (value,)) from None
        key = key.strip()
        if key:
            try:
                widths[image_name(check_sigmas(float(key))[0])] = bw
            except (TypeError, ValueError):
                raise ValueError("%r is not a sigma in mm" % (key,)) from None
        elif default is None and not widths:
            default = bw
        else:
            raise ValueError("%r: only the first entry may be a default bin width" % (spec,))
    if default is not None:
        widths = dict({image_name(s): default for s in sigmas}, **widths)
    return check_bin_widths(widths, sigmas)


@dataclass(frozen=True)
class LineCoefficients:
    """The coefficients of one line filter: n = (N0..N3), m = (M1..M4), d = (D1..D4), bn = (BN1..BN4), bm = (BM1..BM4)."""
    n: tuple
    m: tuple
    d: tuple
    bn: tuple
    bm: tuple

    def flat(self):
        """The 20 values in the order of the C struct lm::LogLine: n, m, d, bn, bm."""
        return self.n + self.m + self.d + self.bn + self.bm


def _trig(sd):
    return (math.sin(W1 / sd), math.sin(W2 / sd), math.cos(W1 / sd), math.cos(W2 / sd), math.exp(L1 / sd),
            math.exp(L2 / sd))


def _numerator(a1, b1, a2, b2, sd):
    """-> (N0, N1, N2, N3), SN, DN, EN."""
    S1, S2, C1, C2, E1, E2 = _trig(sd)
    N0 = a1 + a2
    N1 = E2 * (b2 * S2 - (a2 + 2 * a1) * C2)
    N1 = N1 + E1 * (b1 * S1 - (a1 + 2 * a2) * C1)
    N2 = (a1 + a2) * C2 * C1
    N2 = N2 - (b1 * C2 * S1 + b2 * C1 * S2)
    N2 = N2 * (2 * E1 * E2)
    N2 = N2 + (a2 * E1 * E1 + a1 * E2 * E2)
    N3 = E2 * E1 * E1 * (b2 * S2 - a2 * C2)
    N3 = N3 + E1 * E2 * E2 * (b1 * S1 - a1 * C1)
    return (N0, N1, N2, N3), N0 + N1 + N2 + N3, N1 + 2 * N2 + 3 * N3, N1 + 4 * N2 + 9 * N3


def _denominator(sd):
    """-> (D1, D2, D3, D4), SD, DD, ED."""
    S1, S2, C1, C2, E1, E2 = _trig(sd)
    D1 = -2 * E2 * C2 - 2 * E1 * C1
    D2 = 4 * C2 * C1 * E1 * E2 + E1 * E1 + E2 * E2
    D3 = -2 * C1 * E1 * E2 * E2 - 2 * C2 * E2 * E1 * E1
    D4 = E1 * E1 * E2 * E2
    return (D1, D2, D3, D4), 1 + D1 + D2 + D3 + D4, D1 + 2 * D2 + 3 * D3 + 4 * D4, D1 + 4 * D2 + 9 * D3 + 16 * D4


def coefficients(sd, order):
    """The line filter of order 0 (smoothing) or 2 (normalised second derivative) for sd = sigma / spacing samples, in
    Python floats (float64) with the operations in the order of the module docstring; lm_laplacian_of_gaussian_dev
    forms them with the same operations in C++ (the same libm sin, cos and exp)."""
    sd = float(sd)
    D, SD, DD, ED = _denominator(sd)
    N, SN, DN, EN = _numerator(A1[0], B1[0], A2[0], B2[0], sd)
    if order == 0:
        alpha0 = 2 * SN / SD - N[0]
        N = tuple(x / alpha0 for x in N)
    elif order == 2:
        N2, SN2, DN2, EN2 = _numerator(A1[2], B1[2], A2[2], B2[2], sd)
        beta = -(2 * SN2 - SD * N2[0]) / (2 * SN - SD * N[0])
        N = tuple(x2 + beta * x0 for x2, x0 in zip(N2, N))
        SN, DN, EN = SN2 + beta * SN, DN2 + beta * DN, EN2 + beta * EN
        alpha2 = (EN * SD * SD - ED * SN * SD - 2 * DN * DD * SD + 2 * DD * DD * SN) / (SD * SD * SD)
        k = sd * sd / alpha2
        N = tuple(x * k for x in N)
    else:
        raise ValueError("order must be 0 or 2, got %r" % (order,))
    M = (N[1] - D[0] * N[0], N[2] - D[1] * N[0], N[3] - D[2] * N[0], -D[3] * N[0])
    sum_n = N[0] + N[1] + N[2] + N[3]
    sum_m = M[0] + M[1] + M[2] + M[3]
    return LineCoefficients(N, M, D, tuple(d * sum_n / SD for d in D), tuple(d * sum_m / SD for d in D))


def _e(a, b):
    """((a0 b0 + a1 b1) + a2 b2) + a3 b3 of 4 arrays (or scalars) and 4 coefficients, each operation rounded."""
    return ((a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]) + a[3] * b[3]


def line_filter(x, c):
    """The line filter of LineCoefficients `c` along axis 0 of the float64 array `x` (L, ...): one numpy step per sample
    index over all lines."""
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[0]
    n = [np.float64(t) for t in c.n]
    m = [np.float64(t) for t in c.m]
    d = [np.float64(t) for t in c.d]
    bn = [np.float64(t) for t in c.bn]
    bm = [np.float64(t) for t in c.bm]
    out = np.empty_like(x)
    v = x[0]
    xh, yh = [v, v, v], [v, v, v, v]    # x[i-1..i-3], y[i-1..i-4]
    for i in range(L):
        y = _e([x[i]] + xh, n) - _e(yh, [d[k] if i > k else bn[k] for k in range(4)])
        out[i] = y
        xh = [x[i], xh[0], xh[1]]
        yh = [y, yh[0], yh[1], yh[2]]
    w = x[L - 1]
    xa, za = [w, w, w, w], [w, w, w, w]   # x[j+1..j+4], z[j+1..j+4]
    for j in range(L - 1, -1, -1):
        z = _e(xa, m) - _e(za, [d[k] if L - 1 - j > k else bm[k] for k in range(4)])
        out[j] = out[j] + z
        xa = [x[j], xa[0], xa[1], xa[2]]
        za = [z, za[0], za[1], za[2]]
    return out


def axis_filter(v, axis, c):
    """line_filter along array `axis` of the float64 (S, H, W) array `v`."""
    a = np.ascontiguousarray(np.moveaxis(v, axis, 0))
    return np.moveaxis(line_filter(a, c), 0, axis)


# The passes of each term d = x, y, z (array axes 2, 1, 0): order 0 along the other two in x, y, z order, then order 2
TERMS = ((("y", 0), ("z", 0), ("x", 2)), (("x", 0), ("z", 0), ("y", 2)), (("x", 0), ("y", 0), ("z", 2)))
ARRAY_AXIS = {"x": 2, "y": 1, "z": 0}


def log_host(volume, sigma, spacing):
    """The numpy statement of one LoG image: the float64 LaplacianRecursiveGaussian of `volume` (any real dtype, as
    float64) at `sigma` mm with spacing (x, y, z) mm, normalised across scale.  ValueError as LMInferer.log_images."""
    sigma = check_sigmas(sigma)
    if len(sigma) != 1:
        raise ValueError("log_host: one sigma at a time, got %s" % (sigma,))
    sigma = sigma[0]
    spacing = check_spacing(spacing)
    v = np.asarray(volume)
    check_shape(v.shape, spacing, (sigma,))
    v = v.astype(np.float64)
    if not np.all(np.isfinite(v)):
        raise ValueError("log: the volume holds a NaN or +-inf")
    coeff = {(a, o): coefficients(sigma / spacing["xyz".index(a)], o) for a in "xyz" for o in (0, 2)}
    acc = np.float64(0.0)
    for term in TERMS:
        t = v
        for a, o in term:
            t = axis_filter(t, ARRAY_AXIS[a], coeff[(a, o)])
        acc = acc + t
    return acc


@dataclass
class LogFeatures:
    sigmas: tuple                  # mm, in the order of the images
    classes: tuple                 # the computed classes, in the order of FEATURE_CLASSES
    spacing: Optional[tuple]
    voxel_array_shift: int
    gldm_alpha: int
    images: list = field(default_factory=list)   # wavelet.ImageFeatures per sigma, in the order of `sigmas`

    def __getitem__(self, key):
        """The ImageFeatures of an image name ("log-sigma-1-0-mm-3D") or a sigma (1.0)."""
        name = key if isinstance(key, str) else image_name(key)
        for d in self.images:
            if d.name == name:
                return d
        raise KeyError(key)

    @property
    def labels(self):
        """The row labels (those of `statistics`: each label, then "lung")."""
        d = self.images[0]
        return [r.label for r in (d.first_order or d.texture).rows]

    def voxels(self, label):
        d = self.images[0]
        return (d.first_order or d.texture)[label].voxels

    def vector(self, label):
        """The flat feature vector of a row with PyRadiomics' keys, such as log-sigma-1-0-mm-3D_firstorder_Mean, in
        sigma, class and feature order."""
        return image_vector(self.images, self.classes, label)

    def to_dict(self):
        """JSON-ready: the to_dict() of every image's FirstOrderFeatures and TextureFeatures (NaN as None)."""
        return {"sigmas": list(self.sigmas), "classes": list(self.classes),
                "spacing": list(self.spacing) if self.spacing is not None else None,
                "voxel_array_shift": self.voxel_array_shift, "gldm_alpha": self.gldm_alpha,
                "images": {d.name: d.to_dict() for d in self.images}}
