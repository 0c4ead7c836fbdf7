"""GLCM, GLSZM, GLRLM, GLDM and NGTDM texture features per lung and lobe: the result of LMInferer.texture
(lm_texture_levels_dev, lm_glcm_dev, lm_zone_sizes_dev, lm_glrlm_dev, lm_neighbour_counts_dev; DESIGN §4.9).

Every row of `statistics` (each label, then "lung", mask > 0) is discretised with a fixed bin width as PyRadiomics does:
low = bw * floor(min / bw) and level(x) = floor((floor(x) - low) / bw) + 1, so the row's minimum has level 1 and its
maximum level Ng.  The matrices of the level map are counted exactly on the GPU:
  GLCM   for each of the 13 directions d of the 26-neighbourhood, the symmetric co-occurrence matrix of the voxel pairs
         (v, v + d) with both voxels in the row; the features are computed per direction and averaged over the
         directions that have pairs.
  GLSZM  the number of 26-connected zones of equal level per (level, zone size).
  GLRLM  for each of the 13 directions, the number of maximal runs of equal level per (level, run length); the features
         are averaged over the directions.
  GLDM   the number of voxels per (level, number of the 26 neighbours in the row within gldm_alpha levels).
  NGTDM  per level, the voxels that have neighbours in the row and the sum of |level - mean level of the neighbours|.
The feature formulas are those of PyRadiomics (see the *_features functions; the differences are listed in DESIGN
§4.9).  Everything here is pure numpy in float64; the tests apply the same functions to reference matrices.

PyRadiomics' `distances`, `force2D` / `force2Ddimension` and `weightingNorm` settings (Settings, DESIGN §4.18) replace
the 13 directions by the offset set of `offsets`: GLCM uses it, GLDM and NGTDM the neighbourhood +-O (K = 2 |O|
neighbours, matrices (Ng, K + 1)), GLSZM and GLRLM only follow force2D (8-connected zones within planes, the 4 in-plane
directions), and a weighting norm merges the GLCM and GLRLM matrices with spacing-based weights (`weights`).
"""
import itertools
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from .statistics import UNION

MAX_LEVELS = 255
# (dz, dy, dx) over the array axes (0, 1, 2), in the order of lm_glcm_dev's counts
OFFSETS = ((0, 0, 1), (0, 1, -1), (0, 1, 0), (0, 1, 1)) + tuple((1, dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1))

GLCM_FEATURES = ("Autocorrelation", "JointAverage", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast",
                 "Correlation", "DifferenceAverage", "DifferenceEntropy", "DifferenceVariance", "JointEnergy",
                 "JointEntropy", "Imc1", "Imc2", "Idm", "Idmn", "Id", "Idn", "InverseVariance", "MaximumProbability",
                 "SumEntropy", "SumSquares")
GLSZM_FEATURES = ("SmallAreaEmphasis", "LargeAreaEmphasis", "GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized",
                  "SizeZoneNonUniformity", "SizeZoneNonUniformityNormalized", "ZonePercentage", "GrayLevelVariance",
                  "ZoneVariance", "ZoneEntropy", "LowGrayLevelZoneEmphasis", "HighGrayLevelZoneEmphasis",
                  "SmallAreaLowGrayLevelEmphasis", "SmallAreaHighGrayLevelEmphasis", "LargeAreaLowGrayLevelEmphasis",
                  "LargeAreaHighGrayLevelEmphasis")

# GLRLM and GLDM use the GLSZM formulas with runs / dependence sizes in place of zones (glszm_features); these are the
# GLSZM names they take, in the order of GLRLM_FEATURES and GLDM_FEATURES.
GLRLM_FEATURES = ("ShortRunEmphasis", "LongRunEmphasis", "GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized",
                  "RunLengthNonUniformity", "RunLengthNonUniformityNormalized", "RunPercentage", "GrayLevelVariance",
                  "RunVariance", "RunEntropy", "LowGrayLevelRunEmphasis", "HighGrayLevelRunEmphasis",
                  "ShortRunLowGrayLevelEmphasis", "ShortRunHighGrayLevelEmphasis", "LongRunLowGrayLevelEmphasis",
                  "LongRunHighGrayLevelEmphasis")
GLDM_FEATURES = ("SmallDependenceEmphasis", "LargeDependenceEmphasis", "GrayLevelNonUniformity", "DependenceNonUniformity",
                 "DependenceNonUniformityNormalized", "GrayLevelVariance", "DependenceVariance", "DependenceEntropy",
                 "LowGrayLevelEmphasis", "HighGrayLevelEmphasis", "SmallDependenceLowGrayLevelEmphasis",
                 "SmallDependenceHighGrayLevelEmphasis", "LargeDependenceLowGrayLevelEmphasis",
                 "LargeDependenceHighGrayLevelEmphasis")
_GLDM_AS_GLSZM = ("SmallAreaEmphasis", "LargeAreaEmphasis", "GrayLevelNonUniformity", "SizeZoneNonUniformity",
                  "SizeZoneNonUniformityNormalized", "GrayLevelVariance", "ZoneVariance", "ZoneEntropy",
                  "LowGrayLevelZoneEmphasis", "HighGrayLevelZoneEmphasis", "SmallAreaLowGrayLevelEmphasis",
                  "SmallAreaHighGrayLevelEmphasis", "LargeAreaLowGrayLevelEmphasis", "LargeAreaHighGrayLevelEmphasis")
NGTDM_FEATURES = ("Coarseness", "Contrast", "Busyness", "Complexity", "Strength")

CLASSES = ("glcm", "glszm", "glrlm", "gldm", "ngtdm")
DEFAULT_CLASSES = ("glcm", "glszm")
NEIGHBOURS = 27   # the columns of the GLDM / NGTDM matrices: c or W = 0..26 neighbours

_EPS = np.spacing(1)

MAX_DISTANCE = 3   # the voxel maps' radius limit: the neighbourhood +-O holds at most 342 voxels
WEIGHTING_NORMS = ("manhattan", "euclidean", "infinity", "no_weighting")


def offsets(distances=(1,), force2d_dimension=None):
    """The offset set O as a tuple of (dz, dy, dx) over the array axes (0, 1, 2): every offset whose first non-zero
    component is positive and whose Chebyshev norm is in `distances`, without those moving along axis
    `force2d_dimension` (None: 3-D), in lexicographic order.  offsets() is OFFSETS."""
    ds = check_distances(distances)
    a = None if force2d_dimension is None else check_force2d_dimension(force2d_dimension)
    r = range(-MAX_DISTANCE, MAX_DISTANCE + 1)
    return tuple(o for o in itertools.product(r, r, r)
                 if max(abs(c) for c in o) in ds and next(c for c in o if c) > 0 and (a is None or o[a] == 0))


def check_distances(distances):
    """-> the distances as a sorted tuple of distinct ints in 1..3 (duplicates ignored); TypeError for a string, a
    non-collection or a non-integer item, ValueError for an empty collection or an item outside 1..3."""
    if isinstance(distances, (str, bytes)) or not hasattr(distances, "__iter__"):
        raise TypeError("distances must be a collection of integers such as (1, 2, 3), got %r" % (distances,))
    out = set()
    for d in distances:
        if isinstance(d, (bool, np.bool_)) or not isinstance(d, (int, np.integer)):
            raise TypeError("distances: %r is not an integer" % (d,))
        if not 1 <= int(d) <= MAX_DISTANCE:
            raise ValueError("distances: %d is not in 1..%d" % (int(d), MAX_DISTANCE))
        out.add(int(d))
    if not out:
        raise ValueError("distances: at least one distance in 1..%d is needed" % MAX_DISTANCE)
    return tuple(sorted(out))


def check_force2d_dimension(axis):
    """-> the in-plane axis as an int 0, 1 or 2; TypeError / ValueError otherwise."""
    if isinstance(axis, (bool, np.bool_)) or not isinstance(axis, (int, np.integer)):
        raise TypeError("force2d_dimension must be an integer, got %r" % (axis,))
    if int(axis) not in (0, 1, 2):
        raise ValueError("force2d_dimension must be 0, 1 or 2, got %d" % int(axis))
    return int(axis)


@dataclass(frozen=True)
class Settings:
    """PyRadiomics' neighbourhood settings of the texture matrices (DESIGN §4.18); Settings() is the default."""
    distances: tuple = (1,)
    force2d_dimension: Optional[int] = None   # the axis normal to the planes of force2D; None: 3-D
    weighting_norm: Optional[str] = None      # one of WEIGHTING_NORMS; None: features averaged per direction

    def offsets(self):
        """O of GLCM, GLDM and NGTDM."""
        return offsets(self.distances, self.force2d_dimension)

    def run_offsets(self):
        """The directions of GLRLM, which ignores `distances`: the 13 of OFFSETS, or their 4 in-plane ones."""
        return offsets((1,), self.force2d_dimension)

    def default_neighbourhood(self):
        return self.distances == (1,) and self.force2d_dimension is None


def check_settings(distances=(1,), force2d=False, force2d_dimension=0, weighting_norm=None):
    """-> Settings of `texture`'s arguments; TypeError / ValueError for a bad one.  force2d_dimension is checked even
    when force2d is False."""
    ds = check_distances(distances)
    if not isinstance(force2d, (bool, np.bool_)):
        raise TypeError("force2d must be a bool, got %r" % (force2d,))
    axis = check_force2d_dimension(force2d_dimension)
    if weighting_norm is not None and weighting_norm not in WEIGHTING_NORMS:
        raise ValueError("weighting_norm: unknown norm %r (known: %s, or None)" % (weighting_norm, ", ".join(WEIGHTING_NORMS)))
    return Settings(ds, axis if force2d else None, weighting_norm)


def check_weighting_spacing(settings, spacing):
    """ValueError when the settings' weighting norm needs a spacing and `spacing` is None."""
    if settings.weighting_norm not in (None, "no_weighting") and spacing is None:
        raise ValueError("weighting_norm %r needs the voxel spacing; pass spacing= or an image that has one"
                         % settings.weighting_norm)


def weights(offs, norm, spacing):
    """float64 weight per offset of `offs` for the weighting `norm`, with `spacing` (x, y, z) mm paired with the
    axes as PyRadiomics does (s = (z, y, x), axis 0 <-> z): infinity exp(-max_k(|o_k| s_k)^2), euclidean
    exp(-sum_k (|o_k| s_k)^2), manhattan exp(-(sum_k |o_k| s_k)^2), no_weighting 1."""
    if norm == "no_weighting":
        return np.ones(len(offs), np.float64)
    s = np.asarray(spacing, dtype=np.float64)[::-1]
    d = np.abs(np.asarray(offs, dtype=np.float64).reshape(-1, 3)) * s
    if norm == "infinity":
        return np.exp(-np.max(d, axis=1) ** 2)
    if norm == "euclidean":
        return np.exp(-np.sum(d ** 2, axis=1))
    if norm == "manhattan":
        return np.exp(-np.sum(d, axis=1) ** 2)
    raise ValueError("weighting_norm: unknown norm %r" % (norm,))


def check_arguments(bin_width):
    """-> the bin width as a positive int; TypeError / ValueError otherwise."""
    v = bin_width
    if isinstance(v, (bool, np.bool_)) or not (isinstance(v, (int, np.integer)) or
                                               (isinstance(v, (float, np.floating)) and float(v).is_integer())):
        raise TypeError("bin_width must be an integer, got %r" % (v,))
    if int(v) < 1:
        raise ValueError("bin_width must be a positive integer, got %d" % int(v))
    return int(v)


def check_classes(classes):
    """-> the texture classes as a tuple in the order of CLASSES: a non-empty collection of names from CLASSES.
    TypeError for a string or a non-string name, ValueError for an unknown name or an empty collection."""
    if isinstance(classes, (str, bytes)):
        raise TypeError("classes must be a collection of names such as ('glcm', 'glrlm'), got the string %r" % (classes,))
    names = list(classes)
    for c in names:
        if not isinstance(c, str):
            raise TypeError("classes: %r is not a name" % (c,))
        if c not in CLASSES:
            raise ValueError("classes: unknown texture class %r (known: %s)" % (c, ", ".join(CLASSES)))
    if not names:
        raise ValueError("classes: at least one of %s is needed" % ", ".join(CLASSES))
    return tuple(c for c in CLASSES if c in names)


def check_alpha(alpha):
    """-> the GLDM coarseness parameter as a non-negative int; TypeError / ValueError otherwise."""
    if isinstance(alpha, (bool, np.bool_)) or not isinstance(alpha, (int, np.integer)):
        raise TypeError("gldm_alpha must be an integer, got %r" % (alpha,))
    if int(alpha) < 0:
        raise ValueError("gldm_alpha must be a non-negative integer, got %d" % int(alpha))
    return int(alpha)


def discretisation(vmin, vmax, bin_width, row="the ROI"):
    """-> (low, n_levels) of a row whose values span [vmin, vmax]: low = bw * floor(vmin / bw), n_levels = the level of
    vmax.  ValueError for a non-finite bound (named after `row`) or more than 255 levels."""
    if not (math.isfinite(vmin) and math.isfinite(vmax)):
        raise ValueError("texture: %s holds a non-finite value (min %r, max %r)" % (row, vmin, vmax))
    bw = int(bin_width)
    fmin, fmax = math.floor(vmin), math.floor(vmax)
    low = bw * (fmin // bw)
    ng = (fmax - low) // bw + 1
    if ng > MAX_LEVELS:
        wider = max(bw + 1, (fmax - fmin) // (MAX_LEVELS - 1))
        while (fmax - wider * (fmin // wider)) // wider + 1 > MAX_LEVELS:
            wider += 1
        raise ValueError("texture: %s spans %d grey levels at bin width %d (values %g..%g), more than %d; use a larger "
                         "bin width (%d or more)" % (row, ng, bw, vmin, vmax, MAX_LEVELS, wider))
    return int(low), int(ng)


def levels(values, bin_width, low=None):
    """The level of every value (int64): floor((floor(x) - low) / bw) + 1, low = bw * floor(min / bw) by default.  The
    numpy statement of what lm_texture_levels_dev computes; float16 values are taken as float32, NaN is not allowed."""
    v = np.asarray(values)
    f = np.floor(v.astype(np.float64)).astype(np.int64) if v.dtype.kind == "f" else v.astype(np.int64)
    bw = int(bin_width)
    if low is None:
        low = bw * (int(f.min()) // bw)
    return (f - np.int64(low)) // bw + 1


def _glcm_direction(P, ng):
    """The features of one symmetric (ng, ng) co-occurrence matrix with a positive sum."""
    p = P / P.sum()
    lv = np.arange(1, ng + 1, dtype=np.float64)
    i, j = lv[:, None], lv[None, :]
    px = p.sum(axis=1)
    mu = np.sum(lv * px)
    di = lv - mu
    sx2 = np.sum(di ** 2 * px)
    idx = np.arange(ng)
    p_sum = np.bincount(np.add.outer(idx, idx).ravel(), weights=p.ravel(), minlength=2 * ng - 1)     # k = 2..2 ng
    p_diff = np.bincount(np.abs(np.subtract.outer(idx, idx)).ravel(), weights=p.ravel(), minlength=ng)   # k = 0..ng-1
    k = np.arange(ng, dtype=np.float64)
    pxy = np.outer(px, px)
    hx = -np.sum(px * np.log2(px + _EPS))
    hxy = -np.sum(p * np.log2(p + _EPS))
    hxy1 = -np.sum(p * np.log2(pxy + _EPS))
    hxy2 = -np.sum(pxy * np.log2(pxy + _EPS))
    da = np.sum(k * p_diff)
    s = i + j - 2.0 * mu
    f = {
        "Autocorrelation": np.sum(p * i * j),
        "JointAverage": mu,
        "ClusterProminence": np.sum(s ** 4 * p),
        "ClusterShade": np.sum(s ** 3 * p),
        "ClusterTendency": np.sum(s ** 2 * p),
        "Contrast": np.sum((i - j) ** 2 * p),
        "Correlation": 1.0 if sx2 == 0 else np.sum(np.outer(di, di) * p) / sx2,
        "DifferenceAverage": da,
        "DifferenceEntropy": -np.sum(p_diff * np.log2(p_diff + _EPS)),
        "DifferenceVariance": np.sum((k - da) ** 2 * p_diff),
        "JointEnergy": np.sum(p ** 2),
        "JointEntropy": hxy,
        "Imc1": 0.0 if hx == 0 else (hxy - hxy1) / hx,
        "Imc2": 0.0 if hxy2 <= hxy else math.sqrt(1.0 - math.exp(-2.0 * (hxy2 - hxy))),
        "Idm": np.sum(p_diff / (1.0 + k ** 2)),
        "Idmn": np.sum(p_diff / (1.0 + k ** 2 / float(ng) ** 2)),
        "Id": np.sum(p_diff / (1.0 + k)),
        "Idn": np.sum(p_diff / (1.0 + k / float(ng))),
        "InverseVariance": np.sum(p_diff[1:] / k[1:] ** 2),
        "MaximumProbability": p.max(),
        "SumEntropy": -np.sum(p_sum * np.log2(p_sum + _EPS)),
        "SumSquares": sx2,
    }
    return {name: float(f[name]) for name in GLCM_FEATURES}


def glcm_features(U, n_levels, weights=None):
    """The GLCM features of the unordered pair counts U (|O|, n_levels (n_levels + 1) / 2) in np.triu_indices order:
    per offset P = U + U^T (P(i, i) = 2 U(i, i)), the features of P / sum(P), then the mean over the offsets with
    pairs.  With `weights` (one per offset, see `weights`) the features of the one matrix sum_o w_o P_o instead, summed
    in offset order in float64.  All NaN when there is no pair."""
    ng = int(n_levels)
    U = np.asarray(U, dtype=np.int64).reshape(-1, ng * (ng + 1) // 2)
    iu, ju = np.triu_indices(ng)
    per = []
    merged = np.zeros((ng, ng), np.float64)
    for o, u in enumerate(U):
        if weights is None and not u.any():
            continue
        P = np.zeros((ng, ng), np.float64)
        P[iu, ju] += u
        P[ju, iu] += u
        if weights is None:
            per.append(_glcm_direction(P, ng))
        else:
            merged += weights[o] * P
    if weights is not None and merged.sum() > 0:
        return _glcm_direction(merged, ng)
    if not per:
        return {name: float("nan") for name in GLCM_FEATURES}
    return {name: float(np.mean([f[name] for f in per])) for name in GLCM_FEATURES}


def glszm_features(levels, sizes, counts, n_voxels):
    """The GLSZM features of the zones given as (level, size, count) triples (count zones of `size` voxels at `level`,
    each (level, size) once) of an ROI of n_voxels voxels.  All NaN without zones."""
    c = np.asarray(counts, dtype=np.float64)
    nz = c.sum()
    if nz == 0:
        return {name: float("nan") for name in GLSZM_FEATURES}
    lev = np.asarray(levels, dtype=np.int64)
    sz = np.asarray(sizes, dtype=np.int64)
    i, s = lev.astype(np.float64), sz.astype(np.float64)
    p = c / nz
    by_level = np.bincount(np.unique(lev, return_inverse=True)[1], weights=c)
    by_size = np.bincount(np.unique(sz, return_inverse=True)[1], weights=c)
    mu_i, mu_s = np.sum(p * i), np.sum(p * s)
    f = {
        "SmallAreaEmphasis": np.sum(c / s ** 2) / nz,
        "LargeAreaEmphasis": np.sum(c * s ** 2) / nz,
        "GrayLevelNonUniformity": np.sum(by_level ** 2) / nz,
        "GrayLevelNonUniformityNormalized": np.sum(by_level ** 2) / nz ** 2,
        "SizeZoneNonUniformity": np.sum(by_size ** 2) / nz,
        "SizeZoneNonUniformityNormalized": np.sum(by_size ** 2) / nz ** 2,
        "ZonePercentage": nz / float(n_voxels),
        "GrayLevelVariance": np.sum(p * (i - mu_i) ** 2),
        "ZoneVariance": np.sum(p * (s - mu_s) ** 2),
        "ZoneEntropy": -np.sum(p * np.log2(p + _EPS)),
        "LowGrayLevelZoneEmphasis": np.sum(c / i ** 2) / nz,
        "HighGrayLevelZoneEmphasis": np.sum(c * i ** 2) / nz,
        "SmallAreaLowGrayLevelEmphasis": np.sum(c / (i ** 2 * s ** 2)) / nz,
        "SmallAreaHighGrayLevelEmphasis": np.sum(c * i ** 2 / s ** 2) / nz,
        "LargeAreaLowGrayLevelEmphasis": np.sum(c * s ** 2 / i ** 2) / nz,
        "LargeAreaHighGrayLevelEmphasis": np.sum(c * i ** 2 * s ** 2) / nz,
    }
    return {name: float(f[name]) for name in GLSZM_FEATURES}


def glrlm_features(counts, weights=None):
    """The GLRLM features of the run counts (D, Ng, L) int64 of lm_glrlm_dev (runs of level i + 1 and length k + 1
    along direction d): per direction the GLSZM formulas with runs for zones and lengths for sizes, Nr = the runs and
    Np = sum k P_d(i, k) (the ROI voxels), then the mean over the directions with runs.  With `weights` (one per
    direction) the features of the one matrix sum_d w_d P_d instead, summed in direction order in float64, with Np =
    sum k of that matrix.  All NaN without runs."""
    P = np.asarray(counts, dtype=np.int64)
    if weights is not None:
        merged = np.zeros(P.shape[1:], np.float64)
        for d, p in enumerate(P):
            merged += weights[d] * p
        i, k = np.nonzero(merged)
        if i.size == 0:
            return {name: float("nan") for name in GLRLM_FEATURES}
        c = merged[i, k]
        f = glszm_features(i + 1, k + 1, c, float(np.sum((k + 1) * c)))
        return dict(zip(GLRLM_FEATURES, (f[g] for g in GLSZM_FEATURES)))
    per = []
    for p in P:
        i, k = np.nonzero(p)
        if i.size == 0:
            continue
        c = p[i, k]
        f = glszm_features(i + 1, k + 1, c, int(np.sum((k + 1) * c)))
        per.append(dict(zip(GLRLM_FEATURES, (f[g] for g in GLSZM_FEATURES))))
    if not per:
        return {name: float("nan") for name in GLRLM_FEATURES}
    return {name: float(np.mean([f[name] for f in per])) for name in GLRLM_FEATURES}


def _columns(M):
    """A (Ng, K + 1) neighbour matrix as int64; a flat one is taken as (Ng, 27)."""
    M = np.asarray(M, dtype=np.int64)
    return M if M.ndim == 2 else M.reshape(-1, NEIGHBOURS)


def gldm_features(G):
    """The GLDM features of the dependence counts G (Ng, K + 1) int64 of lm_neighbour_counts_dev (K = 26) or
    lm_neighbour_offsets_dev (voxels of level i + 1 with c neighbours within alpha): the GLSZM formulas with dependence
    size j = c + 1 for the zone size and Nz = sum G = Np.  All NaN without voxels."""
    G = _columns(G)
    i, c = np.nonzero(G)
    f = glszm_features(i + 1, c + 1, G[i, c], int(G.sum()))
    return dict(zip(GLDM_FEATURES, (f[g] for g in _GLDM_AS_GLSZM)))


def ngtdm_features(N, A):
    """The NGTDM features of the counts N (Ng, K + 1) and sums A (Ng, K + 1) int64 of lm_neighbour_counts_dev (K = 26)
    or lm_neighbour_offsets_dev (voxels of level i + 1 with W neighbours in the ROI, and the sum of |W (i + 1) - S| over
    them).  Voxels without neighbours are left out: n_i = sum_{W >= 1} N(i, W), s_i = sum_{W >= 1} A(i, W) / W
    (math.fsum), Nvp = sum n_i, p_i = n_i / Nvp; the sums run over the Ngp levels with p_i > 0.  All NaN when Nvp = 0."""
    N, A = _columns(N), _columns(A)
    n = N[:, 1:].sum(axis=1)
    nvp = int(n.sum())
    if nvp == 0:
        return {name: float("nan") for name in NGTDM_FEATURES}
    keep = np.nonzero(n)[0]
    i = (keep + 1).astype(np.float64)
    p = n[keep] / float(nvp)
    s = np.array([math.fsum(float(A[l, w]) / w for w in range(1, A.shape[1])) for l in keep])
    ngp = keep.size
    ps = p * s
    sum_ps, sum_s = np.sum(ps), np.sum(s)
    dist = np.abs(i[:, None] - i[None, :])
    d2 = dist ** 2
    ip = i * p
    busy = np.sum(np.abs(ip[:, None] - ip[None, :]))
    f = {
        "Coarseness": 1e6 if sum_ps == 0 else 1.0 / sum_ps,
        "Contrast": 0.0 if ngp == 1 else np.sum(p[:, None] * p[None, :] * d2) / (ngp * (ngp - 1)) * sum_s / nvp,
        "Busyness": 0.0 if busy == 0 else sum_ps / busy,
        "Complexity": np.sum(dist * (ps[:, None] + ps[None, :]) / (p[:, None] + p[None, :])) / nvp,
        "Strength": 0.0 if sum_s == 0 else np.sum((p[:, None] + p[None, :]) * d2) / sum_s,
    }
    return {name: float(f[name]) for name in NGTDM_FEATURES}


def runs_from_counts(counts):
    """(k, 4) int64 (direction, level, length, count) rows of the non-zero run counts (13, Ng, L), sorted."""
    P = np.asarray(counts, dtype=np.int64)
    d, i, k = np.nonzero(P)
    return np.stack([d, i + 1, k + 1, P[d, i, k]], axis=1).astype(np.int64).reshape(-1, 4)


def _json_value(v):
    return None if isinstance(v, float) and math.isnan(v) else v


@dataclass
class TextureRow:
    label: object              # the label value (int), or "lung" for the union of all labels
    name: str
    voxels: int                # the ROI: the row's voxels with a non-NaN value
    low: Optional[int]         # bin_width * floor(min / bin_width); None without voxels
    bin_width: int
    n_levels: int              # Ng, the level of the row's maximum; 0 without voxels
    # The feature dicts of a class that was not computed are None.
    glcm: Optional[dict] = field(default_factory=dict)    # GLCM_FEATURES -> float (NaN without pairs)
    glszm: Optional[dict] = field(default_factory=dict)   # GLSZM_FEATURES -> float (NaN without voxels)
    glcm_counts: np.ndarray = field(default_factory=lambda: np.zeros((len(OFFSETS), 0), np.int64))   # U, (|O|, T) int64
    zones: np.ndarray = field(default_factory=lambda: np.zeros((0, 3), np.int64))   # (level, size, count) int64 triples
    glrlm: Optional[dict] = None   # GLRLM_FEATURES -> float (NaN without voxels)
    gldm: Optional[dict] = None    # GLDM_FEATURES -> float (NaN without voxels)
    ngtdm: Optional[dict] = None   # NGTDM_FEATURES -> float (NaN without a voxel that has a neighbour in the ROI)
    # (direction, level, length, count) int64 rows, non-zero, sorted; direction indexes Settings.run_offsets()
    glrlm_runs: Optional[np.ndarray] = None
    gldm_counts: Optional[np.ndarray] = None    # G(i, c), (Ng, K + 1) int64, K = 26 by default
    ngtdm_counts: Optional[np.ndarray] = None   # N(i, W), (Ng, K + 1) int64
    ngtdm_sums: Optional[np.ndarray] = None     # A(i, W) = sum |W i - S|, (Ng, K + 1) int64

    SUMMARY = ("label", "name", "voxels", "low", "bin_width", "n_levels")

    def to_dict(self):
        """JSON-ready: NaN becomes None; the keys of a class appear only when it was computed."""
        d = {k: _json_value(getattr(self, k)) for k in self.SUMMARY}
        for cls in CLASSES:
            f = getattr(self, cls)
            if f is not None:
                d[cls] = {k: _json_value(v) for k, v in f.items()}
            if cls == "glszm" and f is not None:
                d["glszm_zones"] = [[int(x) for x in z] for z in self.zones]
            elif cls == "glrlm" and f is not None:
                d["glrlm_runs"] = self.glrlm_runs.tolist()
            elif cls == "gldm" and f is not None:
                d["gldm_counts"] = self.gldm_counts.tolist()
            elif cls == "ngtdm" and f is not None:
                d["ngtdm_counts"] = self.ngtdm_counts.tolist()
                d["ngtdm_sums"] = self.ngtdm_sums.tolist()
        return d


@dataclass
class TextureFeatures:
    spacing: Optional[tuple]   # (x, y, z) mm, or None; the features do not use it
    bin_width: int
    rows: list
    classes: tuple = DEFAULT_CLASSES   # the computed classes, in the order of CLASSES
    gldm_alpha: int = 0
    settings: Settings = Settings()    # distances, force2D and weighting norm (DESIGN §4.18)

    def __getitem__(self, label):
        """The row of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def to_dict(self):
        """JSON-ready: NaN becomes None.  "classes" appears only when they are not DEFAULT_CLASSES, "gldm_alpha" only
        with GLDM; "distances", "force2d_dimension" and "weighting_norm" only when they are not the defaults, and
        "offsets" (O as [dz, dy, dx] lists) only with a non-default neighbourhood."""
        d = {"spacing": list(self.spacing) if self.spacing is not None else None, "bin_width": self.bin_width}
        if tuple(self.classes) != DEFAULT_CLASSES:
            d["classes"] = list(self.classes)
        if "gldm" in self.classes:
            d["gldm_alpha"] = self.gldm_alpha
        st = self.settings
        if st.distances != (1,):
            d["distances"] = list(st.distances)
        if st.force2d_dimension is not None:
            d["force2d_dimension"] = st.force2d_dimension
        if st.weighting_norm is not None:
            d["weighting_norm"] = st.weighting_norm
        if not st.default_neighbourhood():
            d["offsets"] = [list(o) for o in st.offsets()]
        d["rows"] = [r.to_dict() for r in self.rows]
        return d


def zones_from_native(res):
    """(k, 3) int64 (level, size, count) triples from the dict of _native.Engine.zone_sizes_dev."""
    lev = np.repeat(np.arange(256, dtype=np.int64), res["n_pairs"])
    return np.stack([lev, res["sizes"], res["counts"]], axis=1).astype(np.int64)


def build_row(label, name, voxels, bin_width, low=None, n_levels=0, U=None, zones=None, classes=DEFAULT_CLASSES, runs=None,
              neighbours=None, glcm_weights=None, glrlm_weights=None, columns=NEIGHBOURS):
    """The TextureRow of one row from its exact matrices; voxels == 0 gives an empty row with NaN features.  Only the
    `classes` are filled in, from U and zones (GLCM, GLSZM), the run counts `runs` (D, Ng, L) of lm_glrlm_dev's
    directions (GLRLM) and the (G, N, A) `neighbours` (Ng, `columns`) of lm_neighbour_counts_dev or
    lm_neighbour_offsets_dev (GLDM, NGTDM).  glcm_weights / glrlm_weights: the weighted merge of glcm_features /
    glrlm_features, None for the mean over directions."""
    classes = check_classes(classes)
    nan = lambda names: {k: float("nan") for k in names}   # noqa: E731
    lab = UNION if label == 256 else label
    if voxels == 0:
        row = TextureRow(lab, name, 0, None, int(bin_width), 0, nan(GLCM_FEATURES), nan(GLSZM_FEATURES))
        empty = np.zeros((0, columns), np.int64)
        row.glrlm, row.glrlm_runs = nan(GLRLM_FEATURES), np.zeros((0, 4), np.int64)
        row.gldm, row.gldm_counts = nan(GLDM_FEATURES), empty
        row.ngtdm, row.ngtdm_counts, row.ngtdm_sums = nan(NGTDM_FEATURES), empty, empty.copy()
    else:
        row = TextureRow(lab, name, int(voxels), int(low), int(bin_width), int(n_levels))
        if "glcm" in classes:
            row.glcm_counts = np.asarray(U, dtype=np.int64)
            row.glcm = glcm_features(row.glcm_counts, n_levels, glcm_weights)
        if "glszm" in classes:
            row.zones = np.asarray(zones, dtype=np.int64).reshape(-1, 3)
            row.glszm = glszm_features(row.zones[:, 0], row.zones[:, 1], row.zones[:, 2], voxels)
        if "glrlm" in classes:
            row.glrlm_runs = runs_from_counts(runs)
            row.glrlm = glrlm_features(runs, glrlm_weights)
        if "gldm" in classes or "ngtdm" in classes:
            G, N, A = (np.asarray(m, dtype=np.int64).reshape(-1, columns) for m in neighbours)
            row.gldm_counts, row.gldm = G, gldm_features(G)
            row.ngtdm_counts, row.ngtdm_sums, row.ngtdm = N, A, ngtdm_features(N, A)
    for cls in CLASSES:
        if cls not in classes:
            setattr(row, cls, None)
    for cls, fields in (("gldm", ("gldm_counts",)), ("ngtdm", ("ngtdm_counts", "ngtdm_sums")), ("glrlm", ("glrlm_runs",))):
        if cls not in classes:
            for f in fields:
                setattr(row, f, None)
    return row
