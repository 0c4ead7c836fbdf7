"""Per-label lung volume and density statistics: the result of LMInferer.statistics (lm_label_stats_dev, DESIGN §4.6).

One row per label value l (the voxels with mask == l) and one for the whole lung, "lung" (mask > 0): voxel count, volume
in mL when the spacing is known, NaN count, mean / std / min / max HU, HU percentiles (Perc15 by default) and the
fraction of voxels below HU thresholds (LAA-950 by default).  NaN values are excluded from every value statistic; a row
without values has NaN ones.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

UNION = "lung"
_LUNGS = {1: "right lung", 2: "left lung"}
_LOBES = {1: "left upper lobe", 2: "left lower lobe", 3: "right upper lobe", 4: "right middle lobe", 5: "right lower lobe"}
# the label semantics of the released models (the reference's README, "Semantics of output")
_MODEL_LABELS = {"R231": _LUNGS, "R231CovidWeb": _LUNGS, "LTRCLobes": _LOBES, "LTRCLobes_R231": _LOBES}

THRESHOLD_RANGE = (-1024, 3072)


def label_name(modelname, label):
    """The anatomical name of `label` for a released model, else "label <l>"."""
    return _MODEL_LABELS.get(modelname, {}).get(int(label), "label %d" % int(label))


def check_arguments(percentiles, thresholds):
    """-> (percentiles as floats in [0, 100], thresholds as ints in [-1024, 3072]); ValueError / TypeError otherwise."""
    q = tuple(float(x) for x in np.atleast_1d(np.asarray(percentiles, dtype=np.float64)))
    if any(not (0.0 <= x <= 100.0) for x in q):
        raise ValueError("percentiles must lie in [0, 100], got %s" % (q,))
    t_in = np.atleast_1d(np.asarray(thresholds))
    if t_in.size and not (np.issubdtype(t_in.dtype, np.integer) or
                          (np.issubdtype(t_in.dtype, np.floating) and np.all(t_in == np.round(t_in)))):
        raise TypeError("thresholds must be integer HU values, got %s" % (tuple(t_in.tolist()),))
    t = tuple(int(x) for x in t_in)
    lo, hi = THRESHOLD_RANGE
    if any(not (lo <= x <= hi) for x in t):
        raise ValueError("thresholds must lie in [%d, %d], got %s" % (lo, hi, t))
    if len(q) > 64:
        raise ValueError("at most 64 percentiles per call, got %d" % len(q))
    if len(t) > 4097:
        raise ValueError("at most 4097 thresholds per call, got %d" % len(t))
    return q, t


def _key(x):
    return "%g" % x


def _json_value(v):
    return None if isinstance(v, float) and math.isnan(v) else v


@dataclass
class LabelRow:
    label: object              # the label value (int), or "lung" for the union of all labels
    name: str
    voxels: int
    nan_voxels: int
    volume_ml: Optional[float]  # voxels x voxel volume; None without a spacing
    mean_hu: float
    std_hu: float               # population standard deviation (ddof = 0)
    min_hu: float
    max_hu: float
    percentile_hu: dict = field(default_factory=dict)    # q -> numpy.percentile(values, q)
    fraction_below: dict = field(default_factory=dict)   # t -> fraction of the values below t HU

    def to_dict(self):
        d = {k: _json_value(getattr(self, k)) for k in
             ("label", "name", "voxels", "nan_voxels", "volume_ml", "mean_hu", "std_hu", "min_hu", "max_hu")}
        d["percentile_hu"] = {_key(q): _json_value(v) for q, v in self.percentile_hu.items()}
        d["fraction_below"] = {str(t): _json_value(v) for t, v in self.fraction_below.items()}
        return d


@dataclass
class LabelStatistics:
    spacing: Optional[tuple]   # (x, y, z) mm, or None
    percentiles: tuple
    thresholds: tuple
    rows: list

    def __getitem__(self, label):
        """The row of a label value, or of "lung"."""
        for r in self.rows:
            if r.label == label:
                return r
        raise KeyError(label)

    def to_dict(self):
        """JSON-ready: NaN becomes None."""
        return {"spacing": list(self.spacing) if self.spacing is not None else None, "percentiles": list(self.percentiles),
                "thresholds": list(self.thresholds), "rows": [r.to_dict() for r in self.rows]}


def row_from_native(res, r, label, name, voxel_ml, percentiles, thresholds):
    """The LabelRow of row r of the arrays of _native.Engine.label_stats*; voxel_ml = the voxel volume in mm^3 or None."""
    vox, nan = int(res["voxels"][r]), int(res["nan_voxels"][r])
    n = vox - nan
    m = res["moments"][r]
    return LabelRow(
        label=label, name=name, voxels=vox, nan_voxels=nan, volume_ml=vox * voxel_ml / 1000.0 if voxel_ml is not None else None,
        mean_hu=float(m[0]), std_hu=float(m[1]), min_hu=float(m[2]), max_hu=float(m[3]),
        percentile_hu={q: float(res["percentile"][r][k]) for k, q in enumerate(percentiles)},
        fraction_below={t: (float(res["below_count"][r][k]) / n if n else float("nan")) for k, t in enumerate(thresholds)})


def from_native(res, labels, modelname, spacing, percentiles, thresholds):
    """LabelStatistics from the 257-row arrays of _native.Engine.label_stats*: a row for every label in `labels`, then "lung"."""
    voxel_ml = float(np.prod(np.asarray(spacing, dtype=np.float64))) if spacing is not None else None
    rows = [row_from_native(res, r, UNION if r == 256 else r, UNION if r == 256 else label_name(modelname, r), voxel_ml,
                            percentiles, thresholds) for r in sorted(int(x) for x in labels) + [256]]
    return LabelStatistics(tuple(float(s) for s in spacing) if spacing is not None else None, tuple(percentiles),
                           tuple(thresholds), rows)
