"""Size distributions of low-attenuation clusters: the result of LMInferer.laa_clusters (lm_laa_clusters_dev, DESIGN §4.7).

A low-attenuation (LAA) voxel lies inside the mask and below the threshold (-950 HU by default).  Its clusters are the
connected components of the LAA voxels: per label (a cluster never crosses a label boundary) and for the whole lung,
"lung" (all LAA voxels together).  Each row holds the exact size distribution as (size, count) pairs and D, the
exponent of the power law of the cumulative size distribution (Mishima et al., PNAS 1999, 96:8829): a smaller D means
larger, coalesced clusters.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from .statistics import THRESHOLD_RANGE, UNION, label_name

CONNECTIVITIES = (4, 6, 26)


def check_arguments(threshold, connectivity, min_cluster_voxels):
    """-> (threshold, connectivity, min_cluster_voxels) as ints; ValueError / TypeError otherwise."""
    for name, v in (("threshold", threshold), ("connectivity", connectivity), ("min_cluster_voxels", min_cluster_voxels)):
        if isinstance(v, (bool, np.bool_)) or not (isinstance(v, (int, np.integer)) or
                                                   (isinstance(v, (float, np.floating)) and float(v).is_integer())):
            raise TypeError("%s must be an integer, got %r" % (name, v))
    threshold, connectivity, min_cluster_voxels = int(threshold), int(connectivity), int(min_cluster_voxels)
    lo, hi = THRESHOLD_RANGE
    if not lo <= threshold <= hi:
        raise ValueError("threshold must lie in [%d, %d], got %d" % (lo, hi, threshold))
    if connectivity not in CONNECTIVITIES:
        raise ValueError("connectivity must be 4, 6 or 26, got %d" % connectivity)
    if min_cluster_voxels < 1:
        raise ValueError("min_cluster_voxels must be at least 1, got %d" % min_cluster_voxels)
    return threshold, connectivity, min_cluster_voxels


def fit_d(sizes, counts, min_cluster_voxels=1):
    """D of a size distribution: with the distinct sizes s_i >= min_cluster_voxels and Y_i = the number of clusters of
    size >= s_i, minus the least-squares slope of log10 Y_i on log10 s_i (one point per distinct size).  NaN with fewer
    than two points.  This is one convention; binned fits or other cut-offs can be computed from the same pairs."""
    sizes = np.asarray(sizes, dtype=np.int64)
    counts = np.asarray(counts, dtype=np.int64)
    keep = sizes >= min_cluster_voxels
    s, c = sizes[keep], counts[keep]
    if s.size < 2:
        return float("nan")
    order = np.argsort(s)
    s, c = s[order], c[order]
    y = np.cumsum(c[::-1])[::-1]   # clusters of size >= s_i
    x, ly = np.log10(s.astype(np.float64)), np.log10(y.astype(np.float64))
    xm, ym = x.mean(), ly.mean()
    return float(-np.sum((x - xm) * (ly - ym)) / np.sum((x - xm) ** 2))


def _json_value(v):
    return None if isinstance(v, float) and math.isnan(v) else v


@dataclass
class ClusterRow:
    label: object                 # the label value (int), or "lung" for all LAA voxels together
    name: str
    laa_voxels: int
    laa_volume_ml: Optional[float]   # None without a spacing
    clusters: int
    largest_voxels: int           # 0 without clusters
    largest_ml: Optional[float]
    d: float                      # NaN with fewer than two distinct sizes >= min_cluster_voxels
    sizes: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))    # distinct cluster sizes, ascending
    counts: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))   # clusters of each size

    SUMMARY = ("label", "name", "laa_voxels", "laa_volume_ml", "clusters", "largest_voxels", "largest_ml", "d")

    def to_dict(self):
        d = {k: _json_value(getattr(self, k)) for k in self.SUMMARY}
        d["sizes"] = [int(x) for x in self.sizes]
        d["counts"] = [int(x) for x in self.counts]
        return d


@dataclass
class LaaClusters:
    spacing: Optional[tuple]   # (x, y, z) mm, or None
    threshold: int
    connectivity: int
    min_cluster_voxels: int
    rows: list

    def __getitem__(self, label):
        """The row of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def to_dict(self):
        """JSON-ready: NaN becomes None."""
        return {"spacing": list(self.spacing) if self.spacing is not None else None, "threshold": self.threshold,
                "connectivity": self.connectivity, "min_cluster_voxels": self.min_cluster_voxels,
                "rows": [r.to_dict() for r in self.rows]}


def from_native(res, labels, modelname, spacing, threshold, connectivity, min_cluster_voxels):
    """LaaClusters from the arrays of _native.Engine.laa_clusters*: a row for every label in `labels`, then "lung"."""
    voxel_ml = float(np.prod(np.asarray(spacing, dtype=np.float64))) / 1000.0 if spacing is not None else None
    rows = []
    for r in sorted(int(x) for x in labels) + [256]:
        lo, hi = int(res["offsets"][r]), int(res["offsets"][r + 1])
        sizes, counts = res["sizes"][lo:hi].copy(), res["counts"][lo:hi].copy()
        vox = int(res["laa_voxels"][r])
        largest = int(sizes[-1]) if sizes.size else 0
        rows.append(ClusterRow(
            label=UNION if r == 256 else r, name=UNION if r == 256 else label_name(modelname, r), laa_voxels=vox,
            laa_volume_ml=vox * voxel_ml if voxel_ml is not None else None, clusters=int(res["n_clusters"][r]),
            largest_voxels=largest, largest_ml=largest * voxel_ml if voxel_ml is not None else None,
            d=fit_d(sizes, counts, min_cluster_voxels), sizes=sizes, counts=counts))
    return LaaClusters(tuple(float(s) for s in spacing) if spacing is not None else None, int(threshold), int(connectivity),
                       int(min_cluster_voxels), rows)
