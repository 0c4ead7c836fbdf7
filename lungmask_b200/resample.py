"""PyRadiomics' resampling to resampledPixelSpacing (imageoperations.resampleImage with the sitkBSpline or
sitkNearestNeighbor interpolator): the argument checks, the output grid, the numpy statement resample_host and the result
Resampled of LMInferer.resample (lm_bspline_coefficients_dev, lm_resample_dev; DESIGN §4.19).

Axes use ITK's order: d = x, y, z is array axis 2, 1, 0, and spacings are (x, y, z) mm.  The array is taken as given (no
reorientation) and the mask lies on the image's grid.

Grid (PyRadiomics' resampleImage): ms is the input spacing and rs the requested one (an entry of 0 keeps ms_d); lo_d and
size_d are the bounding box of mask > 0, and an axis with size_d == 1 keeps ms_d.  When np.allclose(ms, rs) nothing is
interpolated: the output is the crop [lo - pad, lo + size - 1 + pad] clamped to the array.  Otherwise, with r = ms / rs,
  L = max(floor((lo - 0.5) r - pad), 0),  U = min(ceil((lo + size - 0.5) r + pad), ceil(N r) - 1),  M = U - L + 1,
  start = 0.5 (rs - ms) / ms + L / r,  c(k) = start + k (rs / ms)     (numpy float64, three 1-D tables)
and output voxel (k_z, k_y, k_x) samples the input at the continuous index (c_z(k_z), c_y(k_y), c_x(k_x)).  The new
origin is origin + D (ms * start).

Sampling: a point with c_d < -0.5 or c_d >= N_d - 0.5 on any axis is 0 in the image and the mask.  The mask, and the image
under "nearest", take the voxel floor(c + 0.5) of each axis (clamped to [0, N - 1]).  The "bspline" image is the cubic
B-spline interpolant with mirror boundaries (Unser / Thevenaz): the float64 coefficients of decompose_host, evaluated
with the weights of bspline_weights on the indices floor(c) - 1 .. floor(c) + 2 mirrored with period 2N - 2, summed x
innermost, then y, then z, each sum from +0.0.  Every product and sum is rounded to float64 on its own.  The result has
the input's dtype (cast_host)."""
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

INTERPOLATORS = ("bspline", "nearest")
MAX_VOXELS = 1 << 32

# The cubic B-spline pole and the constants of its recursive filter, formed in float64 as written
Z = math.sqrt(3.0) - 2.0
GAIN = (1.0 - Z) * (1.0 - 1.0 / Z)
INV_Z = 1.0 / Z
ANTI = Z / (Z * Z - 1.0)
HORIZON = 18   # ceil(ln 1e-10 / ln |z|): lines of at least 19 voxels start from a truncated causal sum
SIXTH = 1.0 / 6.0


def check_interpolator(interpolator):
    if interpolator not in INTERPOLATORS:
        raise ValueError("resample: unknown interpolator %r (known: %s)" % (interpolator, ", ".join(INTERPOLATORS)))
    return interpolator


def check_pad(pad_distance):
    if isinstance(pad_distance, (bool, np.bool_)) or not isinstance(pad_distance, (int, np.integer)) or pad_distance < 0:
        raise ValueError("resample: pad_distance must be a non-negative integer, got %r" % (pad_distance,))
    return int(pad_distance)


def _triple(values, what):
    try:
        sp = tuple(float(s) for s in values)
    except (TypeError, ValueError):
        raise ValueError("resample: %s must be 3 sizes (x, y, z) in mm, got %r" % (what, values)) from None
    if len(sp) != 3 or not all(math.isfinite(s) for s in sp):
        raise ValueError("resample: %s must be 3 finite sizes (x, y, z) in mm, got %r" % (what, values))
    return sp


def check_spacing(spacing):
    """The input spacing (x, y, z): 3 finite positive sizes in mm."""
    if spacing is None:
        raise ValueError("resample: the image spacing is needed; pass spacing=(x, y, z) in mm, a Volume or a SimpleITK image")
    sp = _triple(spacing, "spacing")
    if min(sp) <= 0:
        raise ValueError("resample: spacing must be 3 finite positive sizes (x, y, z) in mm, got %r" % (spacing,))
    return sp


def check_resampled_spacing(resampled_spacing):
    """The requested spacing (x, y, z): 3 finite non-negative sizes in mm (0 keeps the input's along that axis)."""
    sp = _triple(resampled_spacing, "resampled_spacing")
    if min(sp) < 0:
        raise ValueError("resample: resampled_spacing must be 3 finite non-negative sizes (x, y, z) in mm, got %r"
                         % (resampled_spacing,))
    return sp


def parse_spacing(spec):
    """The spacing of a command-line SPEC "X,Y,Z" in mm -> check_resampled_spacing of it; ValueError when malformed."""
    parts = [p.strip() for p in str(spec).split(",")]
    try:
        values = [float(p) for p in parts]
    except ValueError:
        raise ValueError("%r is not three numbers X,Y,Z in mm" % (spec,)) from None
    if len(values) != 3:
        raise ValueError("%r is not three numbers X,Y,Z in mm" % (spec,))
    return check_resampled_spacing(values)


def check_shape(shape, what="the volume"):
    shape = tuple(int(s) for s in shape)
    if len(shape) != 3:
        raise ValueError("resample: expected a (slices, H, W) volume, got shape %s" % (shape,))
    if min(shape) < 1:
        raise ValueError("resample: shape %s is empty" % (shape,))
    if math.prod(shape) >= MAX_VOXELS:
        raise ValueError("resample: %s has shape %s, 2^32 voxels or more" % (what, shape))
    return shape


def bounding_box(mask):
    """(lo, size) of mask > 0, each (x, y, z); ValueError for an empty mask."""
    nz = np.asarray(mask) > 0
    if not nz.any():
        raise ValueError("resample: the mask is empty (no voxel > 0)")
    lo, size = [], []
    for axis in (2, 1, 0):
        hit = np.flatnonzero(nz.any(axis=tuple(a for a in range(3) if a != axis)))
        lo.append(int(hit[0]))
        size.append(int(hit[-1] - hit[0] + 1))
    return tuple(lo), tuple(size)


def bounding_box_of_counts(counts_xyz):
    """bounding_box from the per-plane counts of mask > 0 along x, y and z (lm_plane_label_counts_dev's column 256)."""
    lo, size = [], []
    for c in counts_xyz:
        hit = np.flatnonzero(np.asarray(c) > 0)
        if not hit.size:
            raise ValueError("resample: the mask is empty (no voxel > 0)")
        lo.append(int(hit[0]))
        size.append(int(hit[-1] - hit[0] + 1))
    return tuple(lo), tuple(size)


@dataclass
class Grid:
    crop: bool          # np.allclose(ms, rs): the output is a crop of the input, nothing is interpolated
    spacing: tuple      # the output spacing (x, y, z)
    start: tuple        # the input continuous index (x, y, z) of output voxel 0
    size: tuple         # the output extents (x, y, z)
    tables: tuple       # the float64 continuous-index tables (c_x, c_y, c_z)

    @property
    def shape(self):
        """The output array shape (z, y, x)."""
        return tuple(self.size[::-1])


def grid(shape, spacing, resampled_spacing, lo, size, pad_distance=5):
    """The output grid of an input of array `shape` (z, y, x) and `spacing`, the requested spacing and the mask's bounding
    box (lo, size) (x, y, z) -> Grid.  ValueError when the output has 2^32 voxels or more."""
    pad = check_pad(pad_distance)
    N = np.array(shape[::-1], dtype=np.float64)
    ms = np.array(check_spacing(spacing), dtype=np.float64)
    rs = np.array(check_resampled_spacing(resampled_spacing), dtype=np.float64)
    lo = np.array(lo, dtype=np.float64)
    sz = np.array(size, dtype=np.float64)
    rs = np.where(rs == 0, ms, rs)
    rs = np.where(sz != 1, rs, ms)
    if np.allclose(ms, rs):
        L = np.maximum(lo - pad, 0)
        U = np.minimum(lo + sz - 1 + pad, N - 1)
        M = (U - L + 1).astype(np.int64)
        tables = tuple(L[d] + np.arange(M[d], dtype=np.float64) for d in range(3))
        out = Grid(True, tuple(float(s) for s in ms), tuple(float(x) for x in L), tuple(int(m) for m in M), tables)
    else:
        r = ms / rs
        L = np.floor((lo - 0.5) * r - pad)
        U = np.ceil((lo + sz - 0.5) * r + pad)
        L = np.where(L < 0, 0, L)
        U = np.minimum(U, np.ceil(N * r) - 1)
        M = (U - L + 1).astype(np.int64)
        start = 0.5 * (rs - ms) / ms + L / r
        step = rs / ms
        tables = tuple(start[d] + np.arange(M[d], dtype=np.float64) * step[d] for d in range(3))
        out = Grid(False, tuple(float(s) for s in rs), tuple(float(x) for x in start), tuple(int(m) for m in M), tables)
    if min(out.size) < 1:
        raise ValueError("resample: the output grid %s is empty" % (out.size,))
    if math.prod(out.size) >= MAX_VOXELS:
        raise ValueError("resample: the output grid (x, y, z) %s has 2^32 voxels or more" % (out.size,))
    return out


def new_origin(origin, direction, spacing, start):
    """origin + D (spacing * start): the physical point of output voxel 0 (D row-major 3x3, columns = axes x, y, z)."""
    D = np.asarray(direction, dtype=np.float64).reshape(3, 3)
    return tuple(float(v) for v in np.asarray(origin, np.float64) + D @ (np.asarray(spacing, np.float64)
                                                                        * np.asarray(start, np.float64)))


# ---- the B-spline decomposition --------------------------------------------------------------------------------------

def _initial_causal(c, n):
    """The first causal coefficient of the gain-scaled lines c[0..n-1] (arrays over the other axes)."""
    if n > HORIZON:
        s = c[0].copy()
        zn = Z
        for k in range(1, HORIZON):
            s = s + zn * c[k]
            zn = zn * Z
        return s
    zn = Z
    z2n = Z
    for _ in range(n - 2):
        z2n = z2n * Z   # z^(n-1)
    s = c[0] + z2n * c[n - 1]
    z2n = z2n * (z2n * INV_Z)
    for k in range(1, n - 1):
        s = s + (zn + z2n) * c[k]
        zn = zn * Z
        z2n = z2n * INV_Z
    return s / (1.0 - zn * zn)


def decompose_axis(c, axis):
    """The 1-D cubic B-spline decomposition with mirror boundaries of every line of the float64 array `c` along `axis`
    -> a new array: gain, initial causal coefficient, causal pass, initial anticausal coefficient, anticausal pass.  A
    line of one voxel is left unchanged."""
    a = np.ascontiguousarray(np.moveaxis(np.asarray(c, np.float64), axis, 0)).copy()
    n = a.shape[0]
    if n == 1:
        return np.moveaxis(a, 0, axis)
    a = a * GAIN
    a[0] = _initial_causal(a, n)
    for k in range(1, n):
        a[k] = a[k] + Z * a[k - 1]
    a[n - 1] = ANTI * (Z * a[n - 2] + a[n - 1])
    for k in range(n - 2, -1, -1):
        a[k] = Z * (a[k + 1] - a[k])
    return np.moveaxis(a, 0, axis)


def decompose_host(volume):
    """The float64 B-spline coefficients of the (z, y, x) `volume` (any real dtype, as float64): along x, then y, then z."""
    c = np.asarray(volume).astype(np.float64)
    for axis in (2, 1, 0):
        c = decompose_axis(c, axis)
    return np.ascontiguousarray(c)


# ---- evaluation ------------------------------------------------------------------------------------------------------

def inside(c, n):
    """Whether continuous indices `c` lie in the buffer [-0.5, n - 0.5) of an axis of n voxels."""
    return (c >= -0.5) & (c < n - 0.5)


def nearest_index(c, n):
    """floor(c + 0.5), clamped to [0, n - 1] (int64)."""
    return np.clip(np.floor(c + 0.5), 0, n - 1).astype(np.int64)


def mirror(i, n):
    """Indices `i` mirrored into [0, n) with period 2n - 2 (0 when n == 1)."""
    if n == 1:
        return np.zeros_like(i)
    p = 2 * n - 2
    k = np.mod(i, p)
    return np.where(k >= n, p - k, k)


def bspline_weights(c):
    """(indices (M, 4) before mirroring, weights (M, 4)) of the cubic B-spline at continuous indices `c`."""
    f = np.floor(c)
    w = c - f
    w3 = SIXTH * w * w * w
    w0 = SIXTH + 0.5 * w * (w - 1.0) - w3
    w2 = w + w0 - 2.0 * w3
    w1 = 1.0 - w0 - w2 - w3
    idx = f.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :]
    return idx, np.stack([w0, w1, w2, w3], axis=1)


def _bspline_planes(coeff, tables, planes):
    """The B-spline sum at output planes `planes` (z indices) of the grid `tables` (c_x, c_y, c_z), separably: every
    output voxel's partial sums are the ones the per-voxel 64-tap order forms, so the result is the same bit for bit."""
    n0, n1, n2 = coeff.shape
    (ix, wx), (iy, wy), (iz, wz) = (bspline_weights(t) for t in tables)
    ix, iy, iz = mirror(ix, n2), mirror(iy, n1), mirror(iz, n0)
    iz, wz = iz[planes], wz[planes]
    rows = np.unique(iz)
    pos = np.searchsorted(rows, iz)
    C = coeff[rows]
    t1 = np.zeros((len(rows), n1, len(tables[0])))
    for k in range(4):
        t1 = t1 + wx[:, k][None, None, :] * C[:, :, ix[:, k]]
    t2 = np.zeros((len(rows), len(tables[1]), len(tables[0])))
    for k in range(4):
        t2 = t2 + wy[:, k][None, :, None] * t1[:, iy[:, k], :]
    out = np.zeros((len(planes), len(tables[1]), len(tables[0])))
    for k in range(4):
        out = out + wz[:, k][:, None, None] * t2[pos[:, k]]
    return out


def _nearest_planes(raw, tables, planes):
    n0, n1, n2 = raw.shape
    ix, iy = nearest_index(tables[0], n2), nearest_index(tables[1], n1)
    iz = nearest_index(tables[2], n0)[planes]
    return raw[iz][:, iy][:, :, ix]


def _outside(shape, tables, planes):
    n0, n1, n2 = shape
    ok = (inside(tables[2][planes], n0)[:, None, None] & inside(tables[1], n1)[None, :, None]
          & inside(tables[0], n2)[None, None, :])
    return ~ok


def int_bounds(dtype):
    """The float64 clamp bounds of integer `dtype`: its min, and the largest float64 not above its max."""
    info = np.iinfo(dtype)
    hi = float(info.max)
    if hi > info.max:
        hi = float(np.nextafter(hi, -np.inf))
    return float(info.min), hi


def cast_host(values, dtype):
    """float64 `values` in numpy `dtype`: integers clamped to the type's range, then truncated toward zero; float32 and
    float16 rounded to nearest; float64 kept."""
    dtype = np.dtype(dtype)
    v = np.asarray(values, np.float64)
    if dtype.kind in "iu":
        lo, hi = int_bounds(dtype)
        return np.clip(v, lo, hi).astype(dtype)
    if dtype.kind == "f":
        return v.astype(dtype)
    raise TypeError("resample: no output rule for dtype %s" % dtype)


def resample_host(image, mask, spacing, resampled_spacing=(1.0, 1.0, 1.0), interpolator="bspline", pad_distance=5,
                  planes=None, coeff=None):
    """The numpy statement of LMInferer.resample -> (image, mask uint8, Grid).  `image` (z, y, x) of a real dtype;
    `mask` of its shape; `spacing` and `resampled_spacing` (x, y, z) mm.  `planes`: only these output z indices (default
    all).  `coeff`: decompose_host(image), when the caller already has it.  ValueError for a NaN or +-inf in the image,
    an empty mask, mismatched shapes and bad arguments."""
    check_interpolator(interpolator)
    img = np.asarray(image)
    m = np.asarray(mask)
    check_shape(img.shape)
    if m.shape != img.shape:
        raise ValueError("resample: the mask's shape %s differs from the image's %s" % (m.shape, img.shape))
    if img.dtype == np.bool_ or img.dtype.kind not in "iuf":
        raise TypeError("resample: image dtype %s is not supported" % img.dtype)
    if img.dtype.kind == "f" and not np.all(np.isfinite(img)):
        raise ValueError("resample: the image holds a NaN or +-inf")
    g = grid(img.shape, spacing, resampled_spacing, *bounding_box(m), pad_distance)
    planes = np.arange(g.size[2]) if planes is None else np.asarray(planes, np.int64)
    if g.crop or interpolator == "nearest":
        vals = _nearest_planes(img.astype(np.float64), g.tables, planes)
    else:
        vals = _bspline_planes(decompose_host(img) if coeff is None else coeff, g.tables, planes)
    out_mask = _nearest_planes(m.astype(np.uint8), g.tables, planes)
    outside = _outside(img.shape, g.tables, planes)
    vals[outside] = 0.0
    out_mask[outside] = 0
    return cast_host(vals, img.dtype), out_mask, g


@dataclass
class Resampled:
    """The result of LMInferer.resample: the image (the input's kind and dtype) and the uint8 mask on the new grid."""
    image: object
    mask: object
    spacing: tuple                       # (x, y, z) mm
    start: tuple                         # the input continuous index (x, y, z) of output voxel 0
    origin: Optional[tuple] = None       # LPS mm of output voxel 0, when the input had a geometry
    direction: Optional[tuple] = None    # the input's direction cosines, when it had a geometry

    def volume(self):
        """The image as an io.Volume with the new spacing (and the origin and direction, when known)."""
        from .io import Volume
        a = self.image
        if not isinstance(a, np.ndarray):
            a = a.detach().cpu()
            a = (a.float() if str(a.dtype) == "torch.bfloat16" else a).numpy()
        kw = {}
        if self.origin is not None:
            kw["origin"] = tuple(self.origin)
        if self.direction is not None:
            kw["direction"] = tuple(self.direction)
        return Volume(a, tuple(self.spacing), **kw)
