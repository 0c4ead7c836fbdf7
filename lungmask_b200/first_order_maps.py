"""Voxel-based first-order feature maps of one row: the result of LMInferer.first_order_maps (lm_label_stats_dev,
lm_first_order_maps_dev; DESIGN §4.15), PyRadiomics' voxel-based firstorder extraction (voxelBased=True).

Every ROI voxel c (the row's voxels with a non-NaN value) gets the 18 features of first_order.FIRST_ORDER_FEATURES of
its window W(c) = {v inside the array : max_k |v_k - c_k| <= r}: the candidates are W(c) & ROI (masked_kernel) or the
non-NaN voxels of W(c).  Every other voxel holds init_value.  The discretisation region D is the ROI (masked) or the
non-NaN voxels of the ROI's bounding box padded by r (unmasked); its minimum and maximum give low and n_levels as
first_order.plan_row does.

The fixed operation sequence of a window (n candidates, k = 0.. in (dz, dy, dx) ascending order; every product, sum,
quotient and square root rounded on its own; cvt(i) is the correctly rounded float64 of an integer, float(int)):
  order statistics   the candidates sorted; P_q = numpy.percentile's linear method: h = (n - 1) * (q / 100),
                     a, b = the values at floor(h) and floor(h) + 1 (both the last at h >= n - 1, with t = h + 1, else
                     t = h - floor(h)), numpy's _lerp: a + (b - a) t, or b - (b - a)(1 - t) when t >= 0.5.  Median = P50,
                     Minimum / Maximum the ends, Range = Maximum - Minimum, InterquartileRange = P75 - P25.
  band               B = the candidates with P10 <= x <= P90 (float64 compare), n_B of them.
  exact path         (integer volumes with D exact under plan_row's rule) d = x - base, base = D's minimum; the integer
                     power sums S1..S4 and S_B = sum_B d, then m2n = n S2 - S1^2, m3n = n^2 S3 - 3 n S1 S2 + 2 S1^3,
                     m4n = n^3 S4 - 4 n^2 S1 S3 + 6 n S1^2 S2 - 3 S1^4, A = sum |n d - S1|, A_B = sum_B |n_B d - S_B|,
                     E = S2 + 2 a S1 + n a^2 with a = base + voxel_array_shift:
                       Mean = cvt(base n + S1) / n, Variance = cvt(m2n) / n^2,
                       Skewness = (cvt(m3n) / n^3) / (Variance sqrt(Variance)), Kurtosis = cvt(m4n) / cvt(m2n^2)
                       (both 0 when m2n = 0), MeanAbsoluteDeviation = cvt(A) / n^2,
                       RobustMeanAbsoluteDeviation = cvt(A_B) / n_B^2, Energy = cvt(E).
  float path         (everything else) the values widened to float64 with -0.0 read as +0.0; s = sum x, mean = s / n,
                     e = x - mean, m2 = sum e*e, m3 = sum (e*e)*e, m4 = sum (e*e)*(e*e), mean_B = s_B / n_B,
                     E = sum (x + c)^2 with c = float(voxel_array_shift), each sum in candidate order from 0.0:
                       Mean = mean, Variance = m2 / n, Skewness = (m3 / n) / (Variance sqrt(Variance)),
                       Kurtosis = (m4 / n) / (Variance Variance) (both 0 when m2 = 0),
                       MeanAbsoluteDeviation = (sum |x - mean|) / n, RobustMeanAbsoluteDeviation =
                       (sum_B |x - mean_B|) / n_B, Energy = E.
  both               RobustMeanAbsoluteDeviation is NaN when n_B = 0; RootMeanSquared = sqrt(Energy / n);
                     TotalEnergy = ((s_x s_y) s_z) Energy (NaN without a spacing); Entropy = the sum of T[n][h] and
                     Uniformity the sum of (h / n)(h / n) over the window's levels in ascending order, h the count of a
                     level, T = entropy_table (numpy float64, -(p log2(p + eps)) with p = h / n).
maps_host is this sequence in numpy, vectorised over a chunk of ROI voxels; the device maps equal it bit for bit.
"""
import collections
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import first_order as fo
from .statistics import UNION

RADII = (1, 2, 3)
QUANTILES = (0.1, 0.25, 0.5, 0.75, 0.9)   # q / 100 of first_order.PERCENTILES, as numpy.percentile forms them
SHIFT_LIMIT = 1 << 58    # |voxel_array_shift| and, on the exact path, |base + shift| stay below: E < 2^127
_BITS = {f: 1 << k for k, f in enumerate(fo.FIRST_ORDER_FEATURES)}
_EPS = np.spacing(1)


def check_radius(kernel_radius):
    """-> the kernel radius as an int; ValueError outside 1..3."""
    if isinstance(kernel_radius, (bool, np.bool_)) or not isinstance(kernel_radius, (int, np.integer)) \
            or int(kernel_radius) not in RADII:
        raise ValueError("kernel_radius must be 1, 2 or 3, got %r" % (kernel_radius,))
    return int(kernel_radius)


def check_features(features):
    """-> the requested features in the order of FIRST_ORDER_FEATURES: None for all 18, or a collection of names.
    TypeError for a string, ValueError for an unknown name or an empty collection."""
    if features is None:
        return fo.FIRST_ORDER_FEATURES
    if isinstance(features, (str, bytes)):
        raise TypeError("features must be a collection of names such as ('Mean', 'Entropy'), got the string %r" % (features,))
    want = list(features)
    for f in want:
        if f not in _BITS:
            raise ValueError("unknown first-order feature %r; the features are %s" % (f, ", ".join(fo.FIRST_ORDER_FEATURES)))
    if not want:
        raise ValueError("features is empty")
    return tuple(f for f in fo.FIRST_ORDER_FEATURES if f in want)


def check_label(label):
    """-> the row: an int label 1..255, or "lung" (mask > 0); ValueError otherwise."""
    if label == UNION:
        return UNION
    if isinstance(label, (bool, np.bool_)) or not isinstance(label, (int, np.integer)) or not 1 <= int(label) <= 255:
        raise ValueError('label must be a label value 1..255 or "lung", got %r' % (label,))
    return int(label)


def feature_bits(features):
    """The LM_FO_* bit set of lm_first_order_maps_dev of a checked feature tuple."""
    return sum(_BITS[f] for f in features)


def entropy_table(n_max):
    """T[N][h] = -(p log2(p + eps)), p = h / N, for 1 <= h <= N <= n_max, in numpy float64, flattened by N ascending:
    entry (N, h) at N (N - 1) / 2 + h - 1."""
    n = np.concatenate([np.full(k, k, np.float64) for k in range(1, n_max + 1)])
    h = np.concatenate([np.arange(1, k + 1, dtype=np.float64) for k in range(1, n_max + 1)])
    p = h / n
    return -(p * np.log2(p + _EPS))


def int_to_float(v):
    """The device's correctly rounded int -> float64 of a signed integer below 2^127 in magnitude, restated: the top 64
    significant bits with every shifted-out bit ORed into bit 0, rounded to nearest even, scaled by 2^shift.  Equals
    float(v)."""
    v = int(v)
    neg, m = v < 0, abs(v)
    s = max(m.bit_length() - 64, 0)
    top = m >> s
    if s and m & ((1 << s) - 1):
        top |= 1
    r = math.ldexp(float(top), s)   # float() of a 64-bit int rounds to nearest even, as __ull2double_rn
    return -r if neg else r


@dataclass
class MapsPlan:
    """The discretisation and summation mode of one call."""
    voxels: int              # ROI voxels
    low: Optional[int]
    n_levels: int
    exact: bool
    base: int                # exact: D's minimum; 0 otherwise


def plan_maps(d_voxels, vmin, vmax, bin_width, integer, shift, roi_voxels, row="the ROI"):
    """The MapsPlan of a call whose region D has `d_voxels` voxels spanning [vmin, vmax]: first_order.plan_row's rule
    (ValueError for a non-finite value in D or more than 255 levels) and the shift bound (ValueError)."""
    if not d_voxels or not roi_voxels:
        return MapsPlan(int(roi_voxels), None, 0, False, 0)
    p = fo.plan_row(d_voxels, vmin, vmax, 0.0, (0.0,) * 5, bin_width, integer, row)
    a = p.base + shift if p.exact else shift
    if abs(shift) >= SHIFT_LIMIT or abs(a) >= SHIFT_LIMIT:
        raise ValueError("first_order_maps: voxel_array_shift %d puts |minimum + shift| at 2^58 or more; Energy would "
                         "overflow its 128-bit sum" % shift)
    if not -(1 << 62) < p.low < (1 << 62):
        raise ValueError("first_order_maps: %s holds values beyond +-2^62, which cannot be discretised" % row)
    return MapsPlan(int(roi_voxels), p.low, p.n_levels, p.exact, p.base)


@dataclass
class FirstOrderMaps:
    label: object              # the label value, or "lung"
    kernel_radius: int
    masked_kernel: bool
    bin_width: int
    voxel_array_shift: int
    init_value: float
    low: Optional[int]         # None without ROI voxels
    n_levels: int
    exact: bool
    voxels: int                # ROI voxels
    spacing: Optional[tuple]
    maps: dict = field(default_factory=collections.OrderedDict)   # feature -> (S, H, W) float64

    def __getitem__(self, feature):
        return self.maps[feature]

    def numpy(self):
        """A copy whose maps are numpy arrays."""
        m = collections.OrderedDict((k, v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in self.maps.items())
        return FirstOrderMaps(self.label, self.kernel_radius, self.masked_kernel, self.bin_width, self.voxel_array_shift,
                              self.init_value, self.low, self.n_levels, self.exact, self.voxels, self.spacing, m)


def roi_of(volume, mask, label):
    """The ROI of a row: (mask == label or mask > 0) and a non-NaN value."""
    m = np.asarray(mask).view(np.uint8) if np.asarray(mask).dtype == bool else np.asarray(mask)
    roi = m > 0 if label == UNION else m == label
    v = np.asarray(volume)
    if v.dtype.kind == "f":
        roi &= ~np.isnan(v)
    return roi


def region(volume, roi, radius, masked):
    """D as a boolean array: the ROI, or the non-NaN voxels of its bounding box padded by `radius`."""
    if masked or not roi.any():
        return roi
    d = np.zeros_like(roi)
    sl = []
    for ax in range(3):
        idx = np.nonzero(roi.any(axis=tuple(a for a in range(3) if a != ax)))[0]
        sl.append(slice(max(int(idx[0]) - radius, 0), int(idx[-1]) + radius + 1))
    d[tuple(sl)] = True
    v = np.asarray(volume)
    if v.dtype.kind == "f":
        d &= ~np.isnan(v)
    return d


def _values64(volume):
    v = np.asarray(volume)
    if v.dtype.kind == "f":
        return v.astype(np.float64) + 0.0   # -0.0 read as +0.0
    return v


def maps_host(volume, mask, label=UNION, features=None, kernel_radius=1, masked_kernel=True, bin_width=25,
              voxel_array_shift=0, init_value=0.0, spacing=None, slices=None, chunk=8192):
    """The numpy statement of LMInferer.first_order_maps (the module docstring's sequence) -> FirstOrderMaps with numpy
    maps.  `volume` (S, H, W) numeric (float16 as float32), `mask` uint8 / bool.  `slices`: a range of output slices to
    compute (D still comes from the whole volume); the other slices hold init_value."""
    from .texture import check_arguments
    label = check_label(label)
    feats = check_features(features)
    r = check_radius(kernel_radius)
    bw = check_arguments(bin_width)
    shift = fo.check_shift(voxel_array_shift)
    vol = np.asarray(volume)
    if vol.dtype == np.float16:
        vol = vol.astype(np.float32)
    integer = vol.dtype.kind in "iub"
    roi = roi_of(vol, mask, label)
    D = region(vol, roi, r, masked_kernel)
    n_roi, n_d = int(roi.sum()), int(D.sum())
    vmin = vmax = 0.0
    if n_d:
        dv = vol[D]
        vmin, vmax = float(dv.min()), float(dv.max())
    plan = plan_maps(n_d, vmin, vmax, bw, integer, shift, n_roi, "row %s" % label)
    vv = float("nan") if spacing is None else (float(spacing[0]) * float(spacing[1])) * float(spacing[2])
    out = collections.OrderedDict((f, np.full(vol.shape, float(init_value), np.float64)) for f in feats)
    res = FirstOrderMaps(label, r, bool(masked_kernel), bw, shift, float(init_value), plan.low, plan.n_levels, plan.exact,
                         n_roi, None if spacing is None else tuple(float(s) for s in spacing), out)
    if not n_roi:
        return res
    S, H, W = vol.shape
    cand_arr = roi if masked_kernel else (~np.isnan(vol) if vol.dtype.kind == "f" else np.ones(vol.shape, bool))
    x64 = _values64(vol)
    pad_c = np.pad(cand_arr, r, constant_values=False)
    pad_x = np.pad(x64, r, constant_values=0)
    zz, yy, xx = np.nonzero(roi)
    if slices is not None:
        keep = (zz >= slices.start) & (zz < slices.stop)
        zz, yy, xx = zz[keep], yy[keep], xx[keep]
    offs = [(dz, dy, dx) for dz in range(-r, r + 1) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
    T = entropy_table((2 * r + 1) ** 3)
    for c0 in range(0, len(zz), chunk):
        z, y, x = zz[c0:c0 + chunk] + r, yy[c0:c0 + chunk] + r, xx[c0:c0 + chunk] + r
        cand = np.stack([pad_c[z + dz, y + dy, x + dx] for dz, dy, dx in offs], axis=1)
        vals = np.stack([pad_x[z + dz, y + dy, x + dx] for dz, dy, dx in offs], axis=1)
        f = _window_features(vals, cand, plan, bw, shift, vv, T, feats)
        for k, a in f.items():
            out[k][z - r, y - r, x - r] = a
    return res


def _lerp(a, b, t):
    diff = b - a
    r = a + diff * t
    hi = t >= 0.5
    r[hi] = b[hi] - diff[hi] * (1.0 - t[hi])
    return r


def _window_features(vals, cand, plan, bw, shift, vv, T, feats):
    """The features of a chunk of windows: vals (m, K) in the volume's dtype (float64 on the float path), cand (m, K)
    bool, in candidate order."""
    m, K = vals.shape
    n = cand.sum(axis=1).astype(np.int64)
    nf = n.astype(np.float64)
    exact = plan.exact
    if exact:
        d = np.where(cand, vals.astype(np.int64) - np.int64(plan.base), 0)
        key = np.where(cand, d, np.int64(1) << 40)
        srt = np.sort(key, axis=1)
        xs = srt.astype(np.float64) + float(plan.base)      # exact: |x| <= 2^53 (the sorted tail is never read)
    else:
        x = np.where(cand, vals.astype(np.float64), 0.0)
        srt = np.sort(np.where(cand, x, np.inf), axis=1)
        xs = srt
    rows = np.arange(m)
    pct = []
    for q in QUANTILES:
        h = (n - 1).astype(np.float64) * q
        last = h >= (n - 1).astype(np.float64)
        i = np.floor(h).astype(np.int64)
        ia = np.where(last, n - 1, i)
        ib = np.where(last, n - 1, i + 1)
        t = np.where(last, h + 1.0, h - np.floor(h))
        pct.append(_lerp(xs[rows, ia], xs[rows, np.minimum(ib, K - 1)], t))
    p10, p25, p50, p75, p90 = pct
    vmin, vmax = xs[:, 0], xs[rows, n - 1]
    # band membership in candidate order
    xc = (np.where(cand, vals.astype(np.int64), 0).astype(np.float64)) if exact else x
    band = cand & (xc >= p10[:, None]) & (xc <= p90[:, None])
    nb = band.sum(axis=1).astype(np.int64)
    nan = float("nan")
    f = {}
    if exact:
        S1 = d.sum(axis=1)
        S2 = (d * d).sum(axis=1)
        d3 = d * d * d
        S3 = (d3 >> 32).sum(axis=1).astype(object) * (1 << 32) + (d3 & 0xffffffff).sum(axis=1).astype(object)
        d2 = d * d
        ah, al = d2 >> 20, d2 & 0xfffff
        S4 = ((ah * ah).sum(axis=1).astype(object) * (1 << 40) + (2 * ah * al).sum(axis=1).astype(object) * (1 << 20)
              + (al * al).sum(axis=1).astype(object))
        no, S1o, S2o = n.astype(object), S1.astype(object), S2.astype(object)
        m2n = n * S2 - S1 * S1
        m3n = no * no * S3 - 3 * no * S1o * S2o + 2 * S1o ** 3
        m4n = no ** 3 * S4 - 4 * no * no * S1o * S3 + 6 * no * S1o * S1o * S2o - 3 * S1o ** 4
        sb = np.where(band, d, 0).sum(axis=1)
        A = np.where(cand, np.abs(n[:, None] * d - S1[:, None]), 0).sum(axis=1)
        AB = np.where(band, np.abs(nb[:, None] * d - sb[:, None]), 0).sum(axis=1)
        a = plan.base + shift
        E = (S2o + 2 * a * S1o + no * a * a).astype(np.float64)
        mean = (np.int64(plan.base) * n + S1).astype(np.float64) / nf
        var = m2n.astype(np.float64) / (n * n).astype(np.float64)
        sk = np.zeros(m)
        ku = np.zeros(m)
        nz = m2n != 0
        if nz.any():
            sk[nz] = (m3n[nz].astype(np.float64) / (n[nz] ** 3).astype(np.float64)) / (var[nz] * np.sqrt(var[nz]))
            ku[nz] = m4n[nz].astype(np.float64) / (m2n[nz].astype(object) ** 2).astype(np.float64)
        mad = A.astype(np.float64) / (n * n).astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            rmad = np.where(nb > 0, AB.astype(np.float64) / (nb * nb).astype(np.float64), nan)
    else:
        s = np.zeros(m)
        sbs = np.zeros(m)
        for k in range(K):
            s = s + x[:, k]
            sbs = sbs + np.where(band[:, k], x[:, k], 0.0)
        mean = s / nf
        with np.errstate(invalid="ignore", divide="ignore"):
            mb = sbs / nb.astype(np.float64)
        m2, m3, m4, ad, adb, E = (np.zeros(m) for _ in range(6))
        c = float(shift)
        for k in range(K):
            ck = cand[:, k]
            xk = x[:, k]
            e = xk - mean
            e2 = e * e
            m2 = m2 + np.where(ck, e2, 0.0)
            m3 = m3 + np.where(ck, e2 * e, 0.0)
            m4 = m4 + np.where(ck, e2 * e2, 0.0)
            ad = ad + np.where(ck, np.abs(e), 0.0)
            with np.errstate(invalid="ignore"):
                adb = adb + np.where(band[:, k], np.abs(xk - mb), 0.0)
            t = xk + c
            E = E + np.where(ck, t * t, 0.0)
        var = m2 / nf
        sk = np.zeros(m)
        ku = np.zeros(m)
        nz = m2 != 0
        sk[nz] = (m3[nz] / nf[nz]) / (var[nz] * np.sqrt(var[nz]))
        ku[nz] = (m4[nz] / nf[nz]) / (var[nz] * var[nz])
        mad = ad / nf
        with np.errstate(invalid="ignore", divide="ignore"):
            rmad = np.where(nb > 0, adb / nb.astype(np.float64), nan)
    f["10Percentile"], f["90Percentile"], f["Median"] = p10, p90, p50
    f["InterquartileRange"] = p75 - p25
    f["Minimum"], f["Maximum"], f["Range"] = vmin, vmax, vmax - vmin
    f["Mean"], f["Variance"], f["Skewness"], f["Kurtosis"] = mean, var, sk, ku
    f["MeanAbsoluteDeviation"], f["RobustMeanAbsoluteDeviation"] = mad, rmad
    f["Energy"] = E
    f["RootMeanSquared"] = np.sqrt(E / nf)
    f["TotalEnergy"] = vv * E
    if "Entropy" in feats or "Uniformity" in feats:
        if exact:
            fl = xs
        else:
            fl = np.floor(np.where(np.isfinite(xs), xs, 0.0))
        lev = np.where(np.arange(K)[None, :] < n[:, None],
                       (fl.astype(np.int64) - np.int64(plan.low)) // bw + 1, -1)
        ent, uni = np.zeros(m), np.zeros(m)
        start = np.zeros(m, np.int64)
        base_t = n * (n - 1) // 2
        for k in range(K):
            if k:
                start = np.where(lev[:, k] != lev[:, k - 1], k, start)
            end = (k < n) & ((k == n - 1) | (lev[:, min(k + 1, K - 1)] != lev[:, k]))
            h = k + 1 - start
            ent = ent + np.where(end, T[np.where(end, base_t + h - 1, 0)], 0.0)
            p = h.astype(np.float64) / nf
            uni = uni + np.where(end, p * p, 0.0)
        f["Entropy"], f["Uniformity"] = ent, uni
    return {k: f[k] for k in feats}
