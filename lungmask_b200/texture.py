"""GLCM and GLSZM texture features per lung and lobe: the result of LMInferer.texture (lm_texture_levels_dev, lm_glcm_dev,
lm_zone_sizes_dev; DESIGN §4.9).

Every row of `statistics` (each label, then "lung", mask > 0) is discretised with a fixed bin width as PyRadiomics does:
low = bw * floor(min / bw) and level(x) = floor((floor(x) - low) / bw) + 1, so the row's minimum has level 1 and its
maximum level Ng.  Two matrices of the level map are counted exactly on the GPU:
  GLCM   for each of the 13 directions d of the 26-neighbourhood, the symmetric co-occurrence matrix of the voxel pairs
         (v, v + d) with both voxels in the row; the features are computed per direction and averaged over the
         directions that have pairs.
  GLSZM  the number of 26-connected zones of equal level per (level, zone size).
The feature formulas are those of PyRadiomics (see glcm_features / glszm_features; the differences are listed in DESIGN
§4.9).  Everything here is pure numpy in float64; the tests apply the same functions to reference matrices.
"""
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

_EPS = np.spacing(1)


def check_arguments(bin_width):
    """-> the bin width as a positive int; TypeError / ValueError otherwise."""
    v = bin_width
    if isinstance(v, (bool, np.bool_)) or not (isinstance(v, (int, np.integer)) or
                                               (isinstance(v, (float, np.floating)) and float(v).is_integer())):
        raise TypeError("bin_width must be an integer, got %r" % (v,))
    if int(v) < 1:
        raise ValueError("bin_width must be a positive integer, got %d" % int(v))
    return int(v)


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


def glcm_features(U, n_levels):
    """The GLCM features of the unordered pair counts U (13, n_levels (n_levels + 1) / 2) in np.triu_indices order:
    per direction P = U + U^T (P(i, i) = 2 U(i, i)), the features of P / sum(P), then the mean over the directions with
    pairs.  All NaN when no direction has a pair."""
    ng = int(n_levels)
    U = np.asarray(U, dtype=np.int64).reshape(len(OFFSETS), -1)
    iu, ju = np.triu_indices(ng)
    per = []
    for u in U:
        if not u.any():
            continue
        P = np.zeros((ng, ng), np.float64)
        P[iu, ju] += u
        P[ju, iu] += u
        per.append(_glcm_direction(P, ng))
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
    glcm: dict = field(default_factory=dict)    # GLCM_FEATURES -> float (NaN without pairs)
    glszm: dict = field(default_factory=dict)   # GLSZM_FEATURES -> float (NaN without voxels)
    glcm_counts: np.ndarray = field(default_factory=lambda: np.zeros((len(OFFSETS), 0), np.int64))   # U, (13, T) int64
    zones: np.ndarray = field(default_factory=lambda: np.zeros((0, 3), np.int64))   # (level, size, count) int64 triples

    SUMMARY = ("label", "name", "voxels", "low", "bin_width", "n_levels")

    def to_dict(self):
        d = {k: _json_value(getattr(self, k)) for k in self.SUMMARY}
        d["glcm"] = {k: _json_value(v) for k, v in self.glcm.items()}
        d["glszm"] = {k: _json_value(v) for k, v in self.glszm.items()}
        d["glszm_zones"] = [[int(x) for x in z] for z in self.zones]
        return d


@dataclass
class TextureFeatures:
    spacing: Optional[tuple]   # (x, y, z) mm, or None; the features do not use it
    bin_width: int
    rows: list

    def __getitem__(self, label):
        """The row of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def to_dict(self):
        """JSON-ready: NaN becomes None."""
        return {"spacing": list(self.spacing) if self.spacing is not None else None, "bin_width": self.bin_width,
                "rows": [r.to_dict() for r in self.rows]}


def zones_from_native(res):
    """(k, 3) int64 (level, size, count) triples from the dict of _native.Engine.zone_sizes_dev."""
    lev = np.repeat(np.arange(256, dtype=np.int64), res["n_pairs"])
    return np.stack([lev, res["sizes"], res["counts"]], axis=1).astype(np.int64)


def build_row(label, name, voxels, bin_width, low=None, n_levels=0, U=None, zones=None):
    """The TextureRow of one row from its exact matrices; voxels == 0 gives an empty row with NaN features."""
    if voxels == 0:
        return TextureRow(UNION if label == 256 else label, name, 0, None, int(bin_width), 0,
                          {k: float("nan") for k in GLCM_FEATURES}, {k: float("nan") for k in GLSZM_FEATURES})
    U = np.asarray(U, dtype=np.int64)
    zones = np.asarray(zones, dtype=np.int64).reshape(-1, 3)
    return TextureRow(UNION if label == 256 else label, name, int(voxels), int(low), int(bin_width), int(n_levels),
                      glcm_features(U, n_levels), glszm_features(zones[:, 0], zones[:, 1], zones[:, 2], voxels), U, zones)
