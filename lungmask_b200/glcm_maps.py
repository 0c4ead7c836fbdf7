"""Voxel-based GLCM feature maps of one row: the result of LMInferer.glcm_maps (lm_texture_levels_dev,
lm_glcm_maps_dev; DESIGN §4.16), PyRadiomics' voxel-based glcm extraction (voxelBased=True).

The row, ROI, window W(c), candidates and discretisation region D are those of first_order_maps (DESIGN §4.15).  D is
discretised with texture's fixed bin width (low = bw floor(min_D / bw), Ng = D's n_levels, at most 255); the level map
holds each voxel of D's level and 0 elsewhere, so a candidate is a voxel of W(c) with a non-zero level and a centre a
candidate in the row.  For each of the 13 directions d of texture.OFFSETS, the pairs of a window are (v, v + d) with
both voxels candidates of W(c); P_d = C_d + C_d^T and N = sum P_d (twice the pairs).

The fixed operation sequence of one direction with pairs (every product, sum, quotient and square root rounded on its
own; cvt(k) the correctly rounded float64 of an integer; T = first_order_maps.entropy_table(N_max), T[N][h] at
N (N - 1) / 2 + h - 1; i, j, k, s levels, |i - j| and i + j; Px(i) = sum_j P(i, j), Pd(k), Ps(s) the counts of P with
|i - j| = k and i + j = s; eps = 2^-52):
  integers     A = sum i P, Q = sum i^2 P, B = sum i j P, D1 = sum |i - j| P, D2 = sum (i - j)^2 P,
               S2, S3, S4 = sum (i + j)^k P, E = sum P^2, M = max P (every sum exact)
  rational     Autocorrelation cvt(B) / N, JointAverage cvt(A) / N, Contrast cvt(D2) / N, DifferenceAverage cvt(D1) / N,
               SumSquares cvt(N Q - A^2) / N^2, Correlation cvt(N B - A^2) / cvt(N Q - A^2) (1 when N Q = A^2),
               DifferenceVariance cvt(N D2 - D1^2) / N^2, ClusterTendency cvt(N S2 - 4 A^2) / N^2,
               ClusterShade cvt(N^2 S3 - 6 N A S2 + 16 A^3) / N^3,
               ClusterProminence cvt(N^3 S4 - 8 N^2 A S3 + 24 N A^2 S2 - 48 A^4) / N^4, JointEnergy cvt(E) / N^2,
               MaximumProbability cvt(M) / N
  differences  over k ascending with Pd(k) > 0, each sum from 0.0: DifferenceEntropy + T[N][Pd(k)],
               Idm + cvt(Pd(k)) / cvt(N (1 + k^2)), Idmn + cvt(Pd(k) Ng^2) / cvt(N (Ng^2 + k^2)),
               Id + cvt(Pd(k)) / cvt(N (1 + k)), Idn + cvt(Pd(k) Ng) / cvt(N (Ng + k)),
               InverseVariance + cvt(Pd(k)) / cvt(N k^2) (k >= 1)
  sums         SumEntropy = the sum of T[N][Ps(s)] over s ascending with Ps(s) > 0
  cells        over the cells (i, j), i <= j, of P in (i, j) ascending order, with t counted once on the diagonal and as
               2 t (exact) off it: JointEntropy (HXY) + T[N][P(i, j)], and with w = cvt(Px(i) Px(j)) / cvt(N^2):
               h1 + (cvt(P(i, j)) / N) log2(w + eps); HXY1 = -h1
  levels       over the levels i with Px(i) > 0 ascending: HX + T[N][Px(i)]; for each such i, over the levels j >= i
               with Px(j) > 0 ascending, once on the diagonal and twice off it: h2 + w log2(w + eps); HXY2 = -h2
  Imc          Imc1 = (HXY - HXY1) / HX (0 when HX = 0); Imc2 = sqrt(1 - exp(-2 (HXY2 - HXY))) (0 when HXY2 <= HXY)
log2 and exp are log2_fixed and exp_fixed below, fixed sequences of float64 operations; the device runs the same
operations, so its results are bit-identical.  A window's feature is the sum of its directions' values in direction
order from 0.0, divided by the number of directions with pairs; NaN when no direction has one.
maps_host is this sequence in numpy, vectorised over a chunk of ROI voxels; the device maps equal it bit for bit.
"""
import collections
import functools
from dataclasses import dataclass, field
from typing import ClassVar, Optional

import numpy as np

from . import texture as tx
from .first_order_maps import check_label, check_radius, entropy_table, region, roi_of
from .statistics import UNION

FEATURES = tx.GLCM_FEATURES
_BITS = {f: 1 << k for k, f in enumerate(FEATURES)}
EPS = float.fromhex("0x1p-52")

# log2_fixed: x = 2^e m with m in (sqrt(1/2), sqrt(2)], s = (m - 1) / (m + 1), ln m = 2 s + s z p(z), z = s^2,
# p(z) = sum_k 2 / (2 k + 3) z^k (k = 0..9, the atanh series), log2 x = e + ln(m) log2(e)
_SQRT2 = float.fromhex("0x1.6a09e667f3bcdp+0")
_LOG2E = float.fromhex("0x1.71547652b82fep+0")
_LOG_C = tuple(float.fromhex(h) for h in (
    "0x1.5555555555555p-1", "0x1.999999999999ap-2", "0x1.2492492492492p-2", "0x1.c71c71c71c71cp-3",
    "0x1.745d1745d1746p-3", "0x1.3b13b13b13b14p-3", "0x1.1111111111111p-3", "0x1.e1e1e1e1e1e1ep-4",
    "0x1.af286bca1af28p-4", "0x1.8618618618618p-4"))     # 2/3, 2/5, ..., 2/21
# exp_fixed: k = rint(y log2(e)), r = (y - k ln2_hi) - k ln2_lo (k ln2_hi exact), exp(r) by its Taylor polynomial of
# degree 13 in Horner form, times 2^k
_LN2_HI = float.fromhex("0x1.62e42fee00000p-1")
_LN2_LO = float.fromhex("0x1.a39ef35793c76p-33")
_EXP_C = tuple(float.fromhex(h) for h in (
    "0x1.6124613a86d09p-33", "0x1.1eed8eff8d898p-29", "0x1.ae64567f544e4p-26", "0x1.27e4fb7789f5cp-22",
    "0x1.71de3a556c734p-19", "0x1.a01a01a01a01ap-16", "0x1.a01a01a01a01ap-13", "0x1.6c16c16c16c17p-10",
    "0x1.1111111111111p-7", "0x1.5555555555555p-5", "0x1.5555555555555p-3", "0x1.0000000000000p-1",
    "0x1.0000000000000p+0", "0x1.0000000000000p+0"))     # 1/13!, 1/12!, ..., 1/2!, 1, 1
EXP_DOMAIN = (-708.0, 709.0)   # exp_fixed's arguments: 2^k stays a normal number
LOG2_ULP = 4                   # the stated bounds against the exact function (DESIGN §4.16)
EXP_ULP = 2


def log2_fixed(x):
    """log2 of positive finite float64 values (numpy array or scalar) by the module's fixed sequence."""
    x = np.asarray(x, dtype=np.float64)
    sub = x < float.fromhex("0x1p-1022")
    xs = x * np.where(sub, float.fromhex("0x1p54"), 1.0)
    bits = xs.view(np.int64)
    e = ((bits >> 52) & 0x7ff) - 1023 - np.where(sub, 54, 0)
    m = ((bits & ((1 << 52) - 1)) | (1023 << 52)).view(np.float64)
    big = m > _SQRT2
    m = np.where(big, m * 0.5, m)
    e = e + big
    f = m - 1.0
    s = f / (f + 2.0)
    z = s * s
    p = np.full(x.shape, _LOG_C[-1])
    for c in _LOG_C[-2::-1]:
        p = p * z + c
    lnm = (s + s) + (s * z) * p
    return e.astype(np.float64) + lnm * _LOG2E


def exp_fixed(y):
    """exp of float64 values in EXP_DOMAIN (numpy array or scalar) by the module's fixed sequence."""
    y = np.asarray(y, dtype=np.float64)
    k = np.rint(y * _LOG2E)
    r = (y - k * _LN2_HI) - k * _LN2_LO
    p = np.full(y.shape, _EXP_C[0])
    for c in _EXP_C[1:]:
        p = p * r + c
    return p * ((k.astype(np.int64) + 1023) << 52).view(np.float64)


def check_features(features):
    """-> the requested features in the order of texture.GLCM_FEATURES: None for all 22, or a collection of names.
    TypeError for a string, ValueError for an unknown name or an empty collection."""
    if features is None:
        return FEATURES
    if isinstance(features, (str, bytes)):
        raise TypeError("features must be a collection of names such as ('Contrast', 'Idm'), got the string %r" % (features,))
    want = list(features)
    for f in want:
        if f not in _BITS:
            raise ValueError("unknown GLCM feature %r; the features are %s" % (f, ", ".join(FEATURES)))
    if not want:
        raise ValueError("features is empty")
    return tuple(f for f in FEATURES if f in want)


def feature_bits(features):
    """The feature bits of lm_glcm_maps_dev of a checked feature tuple (bit k = GLCM_FEATURES[k])."""
    return sum(_BITS[f] for f in features)


def max_pairs_n(radius):
    """N_max of a radius: twice the pairs of direction (0, 0, 1) in a full window, (2r+1)^2 2r."""
    e = 2 * int(radius) + 1
    return 2 * e * e * (e - 1)


@dataclass
class GLCMMaps:
    FEATURE_CLASS: ClassVar[str] = "glcm"   # the class part of io.save_feature_maps' file names
    label: object              # the label value, or "lung"
    kernel_radius: int
    masked_kernel: bool
    bin_width: int
    init_value: float
    low: Optional[int]         # None without ROI voxels
    n_levels: int
    voxels: int                # ROI voxels
    maps: dict = field(default_factory=collections.OrderedDict)   # feature -> (S, H, W) float64

    def __getitem__(self, feature):
        return self.maps[feature]

    def numpy(self):
        """A copy whose maps are numpy arrays."""
        m = collections.OrderedDict((k, v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in self.maps.items())
        return GLCMMaps(self.label, self.kernel_radius, self.masked_kernel, self.bin_width, self.init_value, self.low,
                        self.n_levels, self.voxels, m)


def level_map(volume, D, bin_width, row="the ROI"):
    """-> (uint8 level map: D's levels, 0 elsewhere; low; n_levels).  texture.discretisation's refusals (ValueError)."""
    vol = np.asarray(volume)
    if vol.dtype == np.float16:
        vol = vol.astype(np.float32)
    out = np.zeros(vol.shape, np.uint8)
    if not D.any():
        return out, None, 0
    dv = vol[D]
    low, ng = tx.discretisation(float(dv.min()), float(dv.max()), bin_width, row)
    out[D] = tx.levels(dv, bin_width, low)
    return out, low, ng


def maps_host(volume, mask, label=UNION, features=None, kernel_radius=1, masked_kernel=True, bin_width=25,
              init_value=0.0, slices=None, chunk=4096):
    """The numpy statement of LMInferer.glcm_maps (the module docstring's sequence) -> GLCMMaps with numpy maps.
    `volume` (S, H, W) numeric, `mask` uint8 / bool.  `slices`: a range of output slices to compute (D still comes from
    the whole volume); the other slices hold init_value."""
    label = check_label(label)
    feats = check_features(features)
    r = check_radius(kernel_radius)
    bw = tx.check_arguments(bin_width)
    vol = np.asarray(volume)
    if vol.dtype == np.float16:
        vol = vol.astype(np.float32)
    roi = roi_of(vol, mask, label)
    D = region(vol, roi, r, masked_kernel)
    lev, low, ng = level_map(vol, D, bw, "glcm_maps: row %s" % label)
    n_roi = int(roi.sum())
    out = collections.OrderedDict((f, np.full(vol.shape, float(init_value), np.float64)) for f in feats)
    res = GLCMMaps(label, r, bool(masked_kernel), bw, float(init_value), low if n_roi else None, ng if n_roi else 0,
                   n_roi, out)
    if not n_roi:
        return res
    pad = np.pad(lev, r)
    zz, yy, xx = np.nonzero(roi)
    if slices is not None:
        keep = (zz >= slices.start) & (zz < slices.stop)
        zz, yy, xx = zz[keep], yy[keep], xx[keep]
    E = 2 * r + 1
    offs = [(dz, dy, dx) for dz in range(-r, r + 1) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
    T = entropy_table(max_pairs_n(r))
    for c0 in range(0, len(zz), chunk):
        z, y, x = zz[c0:c0 + chunk] + r, yy[c0:c0 + chunk] + r, xx[c0:c0 + chunk] + r
        L = np.stack([pad[z + dz, y + dy, x + dx] for dz, dy, dx in offs], axis=1).astype(np.int64)
        f = window_features(L, E, ng, T)
        for k in feats:
            out[k][z - r, y - r, x - r] = f[k]
    return res


@functools.lru_cache(maxsize=None)
def _pair_positions(E):
    """Per direction of texture.OFFSETS: the window positions (a, b) with b = a + d inside the E^3 window."""
    res = []
    for dz, dy, dx in tx.OFFSETS:
        pa, pb = [], []
        for z in range(E):
            for y in range(E):
                for x in range(E):
                    if 0 <= z + dz < E and 0 <= y + dy < E and 0 <= x + dx < E:
                        pa.append((z * E + y) * E + x)
                        pb.append(((z + dz) * E + y + dy) * E + x + dx)
        res.append((np.array(pa), np.array(pb)))
    return res


def _ascending(cnt):
    """The non-zero entries of each row of `cnt` (m, R) in ascending index order -> (index, count, valid), (m, L)."""
    m, R = cnt.shape
    rows, cols = np.nonzero(cnt)          # row-major: ascending columns within a row
    per = np.bincount(rows, minlength=m)
    L = max(int(per.max()) if m else 0, 1)
    slot = np.arange(len(rows)) - np.repeat(np.cumsum(per) - per, per)
    idx = np.full((m, L), R, np.int64)
    c = np.zeros((m, L), np.int64)
    idx[rows, slot] = cols
    c[rows, slot] = cnt[rows, cols]
    return idx, c, idx < R


def _hist(rows, keys, weights, m, R):
    return np.bincount((rows * R + keys).ravel(), weights=weights.ravel(), minlength=m * R).reshape(m, R).astype(np.int64)


def _cvt(a):
    """cvt of an int64 or object (Python int) array: the correctly rounded float64."""
    return np.asarray(a).astype(np.float64)


def _direction(L, pa, pb, ng, T):
    """The 22 features (dict) and the has-pairs flag of one direction for a chunk of windows L (m, K) int64 levels."""
    m = L.shape[0]
    a, b = L[:, pa], L[:, pb]
    v = (a > 0) & (b > 0)
    a, b = np.where(v, a, 0), np.where(v, b, 0)
    n = 2 * v.sum(axis=1).astype(np.int64)
    has = n > 0
    N = np.where(has, n, 1)
    Nf = N.astype(np.float64)
    s = a + b
    A = s.sum(axis=1)
    Q = (a * a + b * b).sum(axis=1)
    B = 2 * (a * b).sum(axis=1)
    D1 = 2 * np.abs(a - b).sum(axis=1)
    D2 = 2 * ((a - b) ** 2).sum(axis=1)
    S2, S3, S4 = (2 * (s ** k).sum(axis=1) for k in (2, 3, 4))
    No, Ao, S2o, S3o, S4o = (x.astype(object) for x in (N, A, S2, S3, S4))
    f = {}
    f["Autocorrelation"] = _cvt(B) / Nf
    f["JointAverage"] = _cvt(A) / Nf
    f["ClusterProminence"] = _cvt(No ** 3 * S4o - 8 * No * No * Ao * S3o + 24 * No * Ao * Ao * S2o - 48 * Ao ** 4) / _cvt(N ** 4)
    f["ClusterShade"] = _cvt(No * No * S3o - 6 * No * Ao * S2o + 16 * Ao ** 3) / _cvt(N ** 3)
    f["ClusterTendency"] = _cvt(N * S2 - 4 * A * A) / _cvt(N * N)
    f["Contrast"] = _cvt(D2) / Nf
    sq = N * Q - A * A
    with np.errstate(invalid="ignore", divide="ignore"):
        f["Correlation"] = np.where(sq == 0, 1.0, _cvt(N * B - A * A) / _cvt(sq))
    f["DifferenceAverage"] = _cvt(D1) / Nf
    f["DifferenceVariance"] = _cvt(N * D2 - D1 * D1) / _cvt(N * N)
    f["SumSquares"] = _cvt(sq) / _cvt(N * N)
    tb = N * (N - 1) // 2 - 1          # T[N][h] at tb + h
    rows = np.repeat(np.arange(m), a.shape[1]).reshape(a.shape)
    w2 = 2 * v.astype(np.int64)
    # differences and sums
    pd = _hist(rows, np.abs(a - b), w2, m, ng)
    ps = _hist(rows, s, w2, m, 2 * ng + 1)
    de, idm, idmn, idd, idn, iv, se = (np.zeros(m) for _ in range(7))
    g2, g = ng * ng, ng
    k_idx, cnt, ok = _ascending(pd)
    for q in range(k_idx.shape[1]):
        k, c, o = k_idx[:, q], cnt[:, q], ok[:, q]
        cf = _cvt(c)
        de = de + np.where(o, T[tb + np.where(o, c, 1)], 0.0)
        idm = idm + np.where(o, cf / _cvt(N * (1 + k * k)), 0.0)
        idmn = idmn + np.where(o, _cvt(c * g2) / _cvt(N * (g2 + k * k)), 0.0)
        idd = idd + np.where(o, cf / _cvt(N * (1 + k)), 0.0)
        idn = idn + np.where(o, _cvt(c * g) / _cvt(N * (g + k)), 0.0)
        with np.errstate(invalid="ignore", divide="ignore"):
            iv = iv + np.where(o & (k >= 1), cf / _cvt(N * k * k), 0.0)
    s_idx, cnt, ok = _ascending(ps)
    for q in range(s_idx.shape[1]):
        se = se + np.where(ok[:, q], T[tb + np.where(ok[:, q], cnt[:, q], 1)], 0.0)
    f["DifferenceEntropy"], f["Idm"], f["Idmn"], f["Id"], f["Idn"], f["InverseVariance"] = de, idm, idmn, idd, idn, iv
    f["SumEntropy"] = se
    # marginals
    px = _hist(rows, a, v.astype(np.int64), m, ng + 1) + _hist(rows, b, v.astype(np.int64), m, ng + 1)
    px[:, 0] = 0
    NN = _cvt(N * N)
    hx, h2 = np.zeros(m), np.zeros(m)
    lv, pc, ok = _ascending(px)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = _cvt(pc[:, :, None] * pc[:, None, :]) / NN[:, None, None]
        t2 = w * log2_fixed(w + EPS)
    for q in range(lv.shape[1]):
        hx = hx + np.where(ok[:, q], T[tb + np.where(ok[:, q], pc[:, q], 1)], 0.0)
        for q2 in range(q, lv.shape[1]):
            t = t2[:, q, q2]
            h2 = h2 + np.where(ok[:, q] & ok[:, q2], t if q2 == q else 2.0 * t, 0.0)
    # cells in (i, j) ascending order: a run of equal keys ends at k
    key = np.where(v, np.minimum(a, b) * 256 + np.maximum(a, b), 1 << 20)
    srt = np.sort(key, axis=1)
    nxt = np.concatenate([srt[:, 1:], np.full((m, 1), -1)], axis=1)
    end = (srt < (1 << 20)) & (nxt != srt)
    pos = np.arange(srt.shape[1])[None, :]
    first = np.concatenate([np.ones((m, 1), bool), srt[:, 1:] != srt[:, :-1]], axis=1)
    start = np.maximum.accumulate(np.where(first, pos, 0), axis=1)
    lo, hi = np.where(end, srt >> 8, 0), np.where(end, srt & 255, 0)
    diag = lo == hi
    U = pos + 1 - start
    P = np.where(end, np.where(diag, 2 * U, U), 0)
    e2 = np.where(diag, P * P, 2 * P * P).sum(axis=1)
    mx = P.max(axis=1)
    tc = T[tb[:, None] + np.where(end, P, 1)]
    ridx = np.arange(m)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        w = _cvt(px[ridx, lo] * px[ridx, hi]) / NN[:, None]
        t1 = (_cvt(P) / Nf[:, None]) * log2_fixed(w + EPS)
    je, h1 = np.zeros(m), np.zeros(m)
    for k in range(srt.shape[1]):
        dk = diag[:, k]
        je = je + np.where(end[:, k], np.where(dk, tc[:, k], 2.0 * tc[:, k]), 0.0)
        h1 = h1 + np.where(end[:, k], np.where(dk, t1[:, k], 2.0 * t1[:, k]), 0.0)
    f["JointEnergy"] = _cvt(e2) / NN
    f["MaximumProbability"] = _cvt(mx) / Nf
    f["JointEntropy"] = je
    hxy1, hxy2 = -h1, -h2
    with np.errstate(invalid="ignore", divide="ignore"):
        f["Imc1"] = np.where(hx == 0.0, 0.0, (je - hxy1) / hx)
    pos = hxy2 > je
    y = np.where(pos, -2.0 * (hxy2 - je), 0.0)
    f["Imc2"] = np.where(pos, np.sqrt(1.0 - exp_fixed(y)), 0.0)   # exp_fixed(y) <= 1 for y <= 0
    return f, has


def window_features(L, E, ng, T):
    """The 22 features (dict of (m,) float64) of a chunk of windows: L (m, E^3) int64 levels in window order, 0 for a
    voxel that is not a candidate (or outside the array)."""
    m = L.shape[0]
    acc = {k: np.zeros(m) for k in FEATURES}
    nd = np.zeros(m, np.int64)
    for pa, pb in _pair_positions(E):
        f, has = _direction(L, pa, pb, ng, T)
        for k in FEATURES:
            acc[k] = acc[k] + np.where(has, f[k], 0.0)
        nd = nd + has
    with np.errstate(invalid="ignore", divide="ignore"):
        return {k: np.where(nd > 0, acc[k] / nd.astype(np.float64), np.nan) for k in FEATURES}
