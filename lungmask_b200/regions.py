"""Regional lung statistics: the result of LMInferer.regional_statistics (DESIGN §4.8).

Every row of `statistics` (each label, and "lung", the union of all labels) is split two ways:

- craniocaudal zones: whole planes along the craniocaudal array axis, `zones` of them per row, zone 0 the most superior.
  zone_by="volume" (default) gives each zone about the same share of the row's voxels, zone_by="height" the same share
  of the row's craniocaudal extent (`zone_of_planes`).  Every row gets its own boundaries.
- depth shells: the distance of a voxel to the lung surface, the outside of the union of all labels (so fissures are
  interior), from LMInferer.surface_distance.  With bounds b_1 < ... < b_m (mm), shell j holds b_j <= depth < b_{j+1}
  (b_0 = 0, b_{m+1} = inf), compared in float32; shell 0 is the rind, shell m the core.

Each zone or shell row carries the full statistics.LabelRow of its voxels.  The per-plane voxel counts of every row
(the craniocaudal volume profile) come with the result.
"""
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

from .statistics import UNION, check_arguments as check_stat_arguments, label_name, row_from_native

ZONE_BY = ("volume", "height")
MAX_CODES = 255   # uint8 region codes 1..255 per map


def check_arguments(zones, zone_by, shells_mm, percentiles, thresholds):
    """-> (zones, zone_by, shells_mm as a tuple of floats, percentiles, thresholds); ValueError / TypeError otherwise."""
    if isinstance(zones, (bool, np.bool_)) or not isinstance(zones, (int, np.integer)):
        raise TypeError("zones must be an integer, got %r" % (zones,))
    zones = int(zones)
    if not 1 <= zones <= MAX_CODES:
        raise ValueError("zones must lie in [1, %d], got %d" % (MAX_CODES, zones))
    if zone_by not in ZONE_BY:
        raise ValueError("zone_by must be 'volume' or 'height', got %r" % (zone_by,))
    shells = tuple(float(x) for x in np.atleast_1d(np.asarray(shells_mm, dtype=np.float64)))
    if any(not (math.isfinite(b) and b > 0.0) for b in shells):
        raise ValueError("shells_mm must be finite positive depths in mm, got %s" % (shells,))
    f32 = [float(np.float32(b)) for b in shells]
    if any(not f32[i] < f32[i + 1] for i in range(len(f32) - 1)):
        raise ValueError("shells_mm must be strictly increasing (as float32), got %s" % (shells,))
    if len(shells) + 1 > MAX_CODES:
        raise ValueError("at most %d shell bounds, got %d" % (MAX_CODES - 1, len(shells)))
    q, t = check_stat_arguments(percentiles, thresholds)
    return zones, zone_by, shells, q, t


def craniocaudal_axis(code):
    """(array axis, superior at the high index?) of an orientation code such as "LPS": image axis c with code[c] in "SI"
    is array axis 2 - c (arrays are indexed z, y, x); the code names the side an axis increases toward."""
    code = code.upper()
    for c in range(3):
        if code[c] in "SI":
            return 2 - c, code[c] == "S"
    raise ValueError("orientation code %r has no craniocaudal axis" % code)


def zone_of_planes(plane_counts, zones, zone_by="volume", superior_high=True):
    """The zone of every plane of one row: plane_counts (n_planes,) = the row's voxels per plane in array order ->
    int64 (n_planes,), -1 outside the row's first..last occupied plane.  With the planes ordered apex to base (from the
    high index down when superior_high), c_i = the voxels of plane i, C_i = the sum over the planes before it, V the
    total and a..b the first and last plane holding the row, plane i goes to zone
      "height": floor(zones * (i - a) / (b - a + 1))
      "volume": min(zones - 1, floor(zones * (2 C_i + c_i) / (2 V)))   (the midpoint of the plane's share of the volume)
    in integer arithmetic.  Zone 0 is the most superior."""
    c = np.asarray(plane_counts, dtype=np.int64).reshape(-1)
    out = np.full(c.size, -1, np.int64)
    ordered = c[::-1] if superior_high else c
    nz = np.flatnonzero(ordered)
    if nz.size == 0:
        return out
    a, b = int(nz[0]), int(nz[-1])
    i = np.arange(a, b + 1, dtype=np.int64)
    if zone_by == "height":
        z = zones * (i - a) // (b - a + 1)
    elif zone_by == "volume":
        ci = ordered[a:b + 1]
        before = np.cumsum(ci) - ci
        total = int(ci.sum())
        z = np.minimum(zones - 1, zones * (2 * before + ci) // (2 * total))
    else:
        raise ValueError("zone_by must be 'volume' or 'height', got %r" % (zone_by,))
    zo = np.full(c.size, -1, np.int64)
    zo[a:b + 1] = z
    out[:] = zo[::-1] if superior_high else zo
    return out


def zone_names(zones):
    """upper / middle / lower for 3 zones, otherwise "zone k of n" (k = 1 .. n, 1 the most superior)."""
    if zones == 3:
        return ["upper", "middle", "lower"]
    return ["zone %d of %d" % (k + 1, zones) for k in range(zones)]


def shell_names(shells_mm):
    """"depth 0-10 mm", ..., "depth >= 10 mm": one per shell, rind first."""
    edges = [0.0] + list(shells_mm)
    names = ["depth %g-%g mm" % (edges[j], edges[j + 1]) for j in range(len(shells_mm))]
    return names + ["depth >= %g mm" % edges[-1]]


def check_code_budget(labels, buckets, what):
    """The per-label map gives each (present label, bucket) its own uint8 code 1..255."""
    if len(labels) * buckets > MAX_CODES:
        raise ValueError("%s: %d labels x %d %s need %d region codes, a uint8 map holds %d"
                         % (what, len(labels), buckets, what, len(labels) * buckets, MAX_CODES))


def zone_luts(labels, label_zones, lung_zones, zones):
    """(per-label LUT, lung LUT) over the planes of the zone axis: label_zones[l] / lung_zones = zone_of_planes results.
    Label i (of `labels`) in zone z gets code 1 + i * zones + z; the lung map's zone z gets code z + 1."""
    n = lung_zones.size
    lut = np.zeros((n, 256), np.uint8)
    for i, l in enumerate(labels):
        z = label_zones[l]
        lut[:, l] = np.where(z >= 0, 1 + i * zones + z, 0)
    lung = np.zeros((n, 256), np.uint8)
    lung[:, 1:] = np.where(lung_zones >= 0, lung_zones + 1, 0)[:, None]
    return lut, lung


def shell_luts(labels, n_shells):
    """(per-label LUT, lung LUT) over the shells: label i in shell j gets code 1 + i * n_shells + j, the lung map's
    shell j code j + 1."""
    lut = np.zeros((n_shells, 256), np.uint8)
    for i, l in enumerate(labels):
        lut[:, l] = 1 + i * n_shells + np.arange(n_shells)
    lung = np.zeros((n_shells, 256), np.uint8)
    lung[:, 1:] = (np.arange(n_shells) + 1)[:, None]
    return lut, lung


def _plane_range(zone_array, z):
    p = np.flatnonzero(zone_array == z)
    return (int(p[0]), int(p[-1])) if p.size else None


@dataclass
class RegionRow:
    label: object                 # the label value (int), or "lung"
    name: str                     # the label's name
    region: str                   # "zone" or "shell"
    index: int                    # zone 0 = most superior; shell 0 = rind
    region_name: str
    planes: Optional[tuple]       # zones: (first, last) array index along the craniocaudal axis; None without planes
    depth_mm: Optional[tuple]     # shells: (lower, upper) bound in mm, upper inf for the core
    stats: object                 # statistics.LabelRow of the region's voxels

    SUMMARY = ("label", "name", "region", "index", "region_name")

    def to_dict(self):
        d = {k: getattr(self, k) for k in self.SUMMARY}
        d["planes"] = list(self.planes) if self.planes is not None else None
        d["depth_mm"] = [self.depth_mm[0], None if math.isinf(self.depth_mm[1]) else self.depth_mm[1]] \
            if self.depth_mm is not None else None
        d["statistics"] = self.stats.to_dict()
        return d


@dataclass
class RegionalStatistics:
    spacing: Optional[tuple]      # (x, y, z) mm, or None
    zone_axis: int                # the craniocaudal array axis
    superior_high: bool           # whether the superior end is at the high index of zone_axis
    zones: int
    zone_by: str
    shells_mm: tuple
    percentiles: tuple
    thresholds: tuple
    rows: list                    # RegionRow: per label (then "lung") its zones, then its shells
    profile: dict                 # label or "lung" -> int64 (n_planes,) voxels per plane along zone_axis, array order

    def row(self, label, region, index):
        """The RegionRow of (label or "lung", "zone" / "shell", index)."""
        for r in self.rows:
            if r.label == label and r.region == region and r.index == index:
                return r
        raise KeyError((label, region, index))

    def to_dict(self):
        """JSON-ready: NaN becomes None, the profile is one list per row."""
        return {"spacing": list(self.spacing) if self.spacing is not None else None, "zone_axis": self.zone_axis,
                "superior_high": self.superior_high, "zones": self.zones, "zone_by": self.zone_by,
                "shells_mm": list(self.shells_mm), "percentiles": list(self.percentiles),
                "thresholds": list(self.thresholds), "rows": [r.to_dict() for r in self.rows],
                "profile": {str(k): [int(x) for x in v] for k, v in self.profile.items()}}


def _empty_stats(q, t):
    return {"voxels": np.zeros(1, np.int64), "nan_voxels": np.zeros(1, np.int64), "moments": np.full((1, 4), np.nan),
            "percentile": np.full((1, len(q)), np.nan), "below_count": np.zeros((1, len(t)), np.int64)}


def build(labels, present, modelname, spacing, counts, zone_axis, superior_high, zones, zone_by, shells_mm, q, t,
          label_zones, lung_zones, zone_res, zone_lung_res, shell_res, shell_lung_res):
    """RegionalStatistics from the engine's results.  labels: every row label (sorted); present: the labels with voxels,
    in code order; counts: (n_planes, 257) plane counts along zone_axis; *_res: the label_stats arrays of the per-label
    and lung maps of each family (shell ones None without shells)."""
    voxel_ml = float(np.prod(np.asarray(spacing, dtype=np.float64))) if spacing is not None else None
    empty = _empty_stats(q, t)
    znames, snames = zone_names(zones), shell_names(shells_mm)
    n_shells = len(shells_mm) + 1
    edges = [0.0] + list(shells_mm) + [math.inf]
    index = {l: i for i, l in enumerate(present)}
    rows, profile = [], {}
    for l in list(labels) + [UNION]:
        lung = l == UNION
        name = UNION if lung else label_name(modelname, l)
        profile[l] = counts[:, 256].copy() if lung else counts[:, l].copy()
        zarr = lung_zones if lung else label_zones.get(l)
        for z in range(zones):
            if lung:
                res, r = zone_lung_res, z + 1
            elif l in index:
                res, r = zone_res, 1 + index[l] * zones + z
            else:
                res, r = empty, 0
            rows.append(RegionRow(l, name, "zone", z, znames[z], _plane_range(zarr, z) if zarr is not None else None, None,
                                  row_from_native(res, r, l, name, voxel_ml, q, t)))
        if shell_res is None:
            continue
        for j in range(n_shells):
            if lung:
                res, r = shell_lung_res, j + 1
            elif l in index:
                res, r = shell_res, 1 + index[l] * n_shells + j
            else:
                res, r = empty, 0
            rows.append(RegionRow(l, name, "shell", j, snames[j], None, (edges[j], edges[j + 1]),
                                  row_from_native(res, r, l, name, voxel_ml, q, t)))
    return RegionalStatistics(tuple(float(s) for s in spacing) if spacing is not None else None, int(zone_axis),
                              bool(superior_high), zones, zone_by, tuple(shells_mm), tuple(q), tuple(t), rows, profile)
