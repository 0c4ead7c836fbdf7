"""PyRadiomics' first-order features per lung and lobe: the result of LMInferer.first_order (lm_label_stats_dev,
lm_first_order_sums_dev, lm_first_order_splits_dev; DESIGN §4.11).

Every row of `statistics` (each label, then "lung", mask > 0) gets the 18 default firstorder features of PyRadiomics
(FIRST_ORDER_FEATURES).  Its ROI is its voxels with a non-NaN value.  The percentiles, the minimum and the maximum come
from one lm_label_stats_dev call (bit-identical to numpy.percentile); the rest from two passes over the volume:
  A  the level histogram of the fixed-bin-width discretisation of texture.discretisation (Entropy, Uniformity) and the
     power sums of the values, over the ROI and over the band P10 <= x <= P90;
  B  the split sums that turn the absolute deviations about the mean (and the band's mean) into sums.
Exact rows (integer volumes whose row spans less than 2^20, see plan_row) are summed in integers about the row's minimum,
d = x - min: S_k = sum d^k, and the features are formed from Python integers and Fractions, each rounded once to float64
in a fixed order, so they are reproducible bit for bit.  Float rows are summed in float64 about the statistics' mean.
"""
import math
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Optional

import numpy as np

from .statistics import UNION
from .texture import discretisation

FIRST_ORDER_FEATURES = ("10Percentile", "90Percentile", "Energy", "Entropy", "InterquartileRange", "Kurtosis", "Maximum",
                        "MeanAbsoluteDeviation", "Mean", "Median", "Minimum", "Range", "RobustMeanAbsoluteDeviation",
                        "RootMeanSquared", "Skewness", "TotalEnergy", "Uniformity", "Variance")
PERCENTILES = (10.0, 25.0, 50.0, 75.0, 90.0)   # the q of the lm_label_stats_dev call, in this order
EXACT_SPAN = 1 << 20        # an exact row spans fewer than 2^20 integer values ...
EXACT_LIMIT = 1 << 53       # ... and its minimum and maximum are exact in float64
MODE_SKIP, MODE_FLOAT, MODE_EXACT = 0, 1, 2   # the row modes of the C calls

_EPS = np.spacing(1)


def check_shift(shift):
    """-> the voxel array shift (PyRadiomics' voxelArrayShift) as an int; TypeError for anything but an integer."""
    if isinstance(shift, (bool, np.bool_)) or not isinstance(shift, (int, np.integer)):
        raise TypeError("voxel_array_shift must be an integer, got %r" % (shift,))
    return int(shift)


@dataclass
class RowPlan:
    """What the passes need of one row: its ROI size, the discretisation and the summation mode."""
    voxels: int
    low: int
    n_levels: int
    exact: bool
    base: int              # exact rows: the integer minimum, the origin of d = x - base; 0 otherwise
    vmin: float
    vmax: float
    mean: float            # the float mean of lm_label_stats_dev: the centre of a float row's pass A
    percentiles: tuple     # P10, P25, P50, P75, P90


def plan_row(voxels, vmin, vmax, mean, percentiles, bin_width, integer, row="the ROI"):
    """The RowPlan of a row of `voxels` ROI voxels with the statistics' min, max, mean and PERCENTILES.  ValueError for a
    non-finite value in the ROI or more than 255 levels (named after `row`).  `integer`: the volume holds integers; the
    row is then exact when max - min < 2^20 and |min|, |max| <= 2^53."""
    try:
        low, ng = discretisation(vmin, vmax, bin_width, row)
    except ValueError as ex:
        raise ValueError("first_order: " + str(ex).split(": ", 1)[1]) from None
    exact = bool(integer) and abs(vmin) <= EXACT_LIMIT and abs(vmax) <= EXACT_LIMIT and int(vmax) - int(vmin) < EXACT_SPAN
    return RowPlan(int(voxels), low, ng, exact, int(vmin) if exact else 0, float(vmin), float(vmax), float(mean),
                   tuple(float(p) for p in percentiles))


def split_points(plan, power_sums, band_count, band_sum):
    """-> (split, split_band): exact rows, floor(S1 / n) and floor(S_B / n_B) (0 without band voxels); float rows, the
    mean and the band's mean (the centre without band voxels)."""
    n, nb = plan.voxels, int(band_count)
    if plan.exact:
        return int(power_sums[0]) // n, (int(band_sum) // nb if nb else 0)
    c = plan.mean
    return c + float(power_sums[0]) / n, (c + float(band_sum) / nb if nb else c)


def sums_host(values, plan, bin_width):
    """The numpy statement of both passes for one row: `values` are its ROI values (no NaN) in the volume's dtype.
    -> (histogram int64 [n_levels], power_sums [4], band_count, band_sum, splits [4] or [2]), with Python ints on an
    exact row and floats on a float row (their sums in numpy's order, not the device's)."""
    v = np.asarray(values).reshape(-1)
    f = np.floor(v.astype(np.float64)).astype(np.int64) if v.dtype.kind == "f" else v.astype(np.int64)
    lev = (f - np.int64(plan.low)) // int(bin_width) + 1
    hist = np.bincount(lev, minlength=plan.n_levels + 1)[1:].astype(np.int64)
    x = v.astype(np.float64)
    band = (x >= plan.percentiles[0]) & (x <= plan.percentiles[4])
    nb = int(band.sum())
    if plan.exact:
        d = v.astype(np.int64) - np.int64(plan.base)
        vals, cnt = np.unique(d, return_counts=True)
        vals, cnt = [int(a) for a in vals], [int(c) for c in cnt]
        S = [sum(c * a ** k for a, c in zip(vals, cnt)) for k in (1, 2, 3, 4)]
        sb = int(d[band].sum())
        t, tb = split_points(plan, S, nb, sb)
        lo, lob = d <= t, band & (d <= tb)
        splits = [int(lo.sum()), int(d[lo].sum()), int(lob.sum()), int(d[lob].sum())]
        return hist, S, nb, sb, splits
    e = x - plan.mean
    S = [float(np.sum(e ** k)) for k in (1, 2, 3, 4)]
    sb = float(np.sum(e[band]))
    mu, mub = split_points(plan, S, nb, sb)
    splits = [float(np.sum(np.abs(x - mu))), float(np.sum(np.abs(x[band] - mub)))]
    return hist, S, nb, sb, splits


def features(plan, histogram, power_sums, band_count, band_sum, splits, spacing=None, shift=0):
    """The 18 features of FIRST_ORDER_FEATURES of a row from its plan and its sums (as sums_host returns them, or as the
    device gives them).  Exact rows are formed in Python integers / Fractions and rounded once each; float rows in
    float64.  TotalEnergy is NaN without a spacing."""
    n, nb = plan.voxels, int(band_count)
    p10, p25, p50, p75, p90 = plan.percentiles
    h = np.asarray(histogram, dtype=np.float64)
    p = h / float(n)
    nan = float("nan")
    if plan.exact:
        S1, S2, S3, S4 = (int(s) for s in power_sums)
        sb = int(band_sum)
        n_lo, L, n_lo_b, L_b = (int(s) for s in splits)
        m2n = n * S2 - S1 * S1                                                 # n^2 m2
        m3n = n * n * S3 - 3 * n * S1 * S2 + 2 * S1 ** 3                       # n^3 m3
        m4n = n ** 3 * S4 - 4 * n * n * S1 * S3 + 6 * n * S1 * S1 * S2 - 3 * S1 ** 4   # n^4 m4
        variance = float(Fraction(m2n, n * n))
        skewness = 0.0 if m2n == 0 else float(Fraction(m3n, n ** 3)) / variance ** 1.5
        kurtosis = 0.0 if m2n == 0 else float(Fraction(m4n, m2n * m2n))
        mean = float(Fraction(plan.base * n + S1, n))
        # sum |d - mu| = (S1 - 2L) + (2 n_lo - n) S1 / n: the voxels with d <= floor(mu) lie at or below mu, the rest above
        mad = float(Fraction(n * (S1 - 2 * L) + (2 * n_lo - n) * S1, n * n))
        rmad = float(Fraction(nb * (sb - 2 * L_b) + (2 * n_lo_b - nb) * sb, nb * nb)) if nb else nan
        a = plan.base + int(shift)
        energy_i = S2 + 2 * a * S1 + n * a * a
        energy = float(energy_i)
        rms = math.sqrt(float(Fraction(energy_i, n)))
    else:
        F1, F2, F3, F4 = (float(s) for s in power_sums)
        c = plan.mean
        dm = F1 / n
        e2, e3, e4 = F2 / n, F3 / n, F4 / n
        m2 = max(e2 - dm * dm, 0.0)
        m3 = e3 - 3.0 * dm * e2 + 2.0 * dm ** 3
        m4 = e4 - 4.0 * dm * e3 + 6.0 * dm * dm * e2 - 3.0 * dm ** 4
        variance = m2
        skewness = 0.0 if m2 == 0 else m3 / m2 ** 1.5
        kurtosis = 0.0 if m2 == 0 else m4 / (m2 * m2)
        mean = c + dm
        mad = float(splits[0]) / n
        rmad = float(splits[1]) / nb if nb else nan
        a = c + float(shift)
        energy = F2 + 2.0 * a * F1 + n * a * a
        rms = math.sqrt(energy / n)
    if spacing is not None:
        sx, sy, sz = (float(s) for s in spacing)
        total = sx * sy * sz * energy
    else:
        total = nan
    f = {
        "10Percentile": p10,
        "90Percentile": p90,
        "Energy": energy,
        "Entropy": float(-np.sum(p * np.log2(p + _EPS))),
        "InterquartileRange": p75 - p25,
        "Kurtosis": kurtosis,
        "Maximum": plan.vmax,
        "MeanAbsoluteDeviation": mad,
        "Mean": mean,
        "Median": p50,
        "Minimum": plan.vmin,
        "Range": plan.vmax - plan.vmin,
        "RobustMeanAbsoluteDeviation": rmad,
        "RootMeanSquared": rms,
        "Skewness": skewness,
        "TotalEnergy": total,
        "Uniformity": float(np.sum(p * p)),
        "Variance": variance,
    }
    return {k: float(f[k]) for k in FIRST_ORDER_FEATURES}


def _json_value(v):
    return None if isinstance(v, float) and math.isnan(v) else v


def _plain(v):
    """A power or split sum as a JSON-ready Python int or float."""
    return int(v) if isinstance(v, (int, np.integer)) else float(v)


@dataclass
class FirstOrderRow:
    label: object              # the label value (int), or "lung" for the union of all labels
    name: str
    voxels: int                # the ROI: the row's voxels with a non-NaN value
    exact: Optional[bool]      # summed exactly in integers (see plan_row); None without voxels
    low: Optional[int]         # bin_width * floor(min / bin_width); None without voxels
    bin_width: int
    n_levels: int              # Ng, the level of the row's maximum; 0 without voxels
    features: dict = field(default_factory=dict)   # FIRST_ORDER_FEATURES -> float (NaN without voxels)
    histogram: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))   # voxels per level 1..Ng, int64
    percentiles: dict = field(default_factory=dict)   # q of PERCENTILES -> the value (numpy.percentile)
    origin: Optional[float] = None   # exact rows: the base (int) of d = x - base; float rows: the centre c of e = x - c
    power_sums: list = field(default_factory=list)    # sum d^k (ints) or sum e^k (floats), k = 1..4
    band_count: int = 0         # the voxels with P10 <= x <= P90
    band_sum: object = 0        # sum d (int) or sum e (float) over them
    splits: list = field(default_factory=list)   # exact: n_lo, L, n_lo_B, L_B; float: sum |x - mu|, sum_B |x - mu_B|

    SUMMARY = ("label", "name", "voxels", "exact", "low", "bin_width", "n_levels")

    def to_dict(self):
        """JSON-ready: NaN becomes None; the sums stay exact Python ints on exact rows."""
        d = {k: _json_value(getattr(self, k)) for k in self.SUMMARY}
        d["features"] = {k: _json_value(v) for k, v in self.features.items()}
        d["histogram"] = [int(x) for x in self.histogram]
        d["percentiles"] = {"%g" % q: _json_value(v) for q, v in self.percentiles.items()}
        d["origin"] = _json_value(self.origin)
        d["power_sums"] = [_plain(s) for s in self.power_sums]
        d["band_count"] = int(self.band_count)
        d["band_sum"] = _plain(self.band_sum)
        d["splits"] = [_plain(s) for s in self.splits]
        return d


@dataclass
class FirstOrderFeatures:
    spacing: Optional[tuple]   # (x, y, z) mm, or None (TotalEnergy is then NaN)
    bin_width: int
    voxel_array_shift: int
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
                "voxel_array_shift": self.voxel_array_shift, "rows": [r.to_dict() for r in self.rows]}


def build_row(label, name, bin_width, plan=None, histogram=None, power_sums=None, band_count=0, band_sum=0, splits=None,
              spacing=None, shift=0):
    """The FirstOrderRow of one row from its plan and sums; plan None gives an empty row with NaN features."""
    lab = UNION if label == 256 else label
    if plan is None:
        return FirstOrderRow(lab, name, 0, None, None, int(bin_width), 0, {k: float("nan") for k in FIRST_ORDER_FEATURES})
    hist = np.asarray(histogram, dtype=np.int64)[:plan.n_levels]
    conv = int if plan.exact else float
    ps = [conv(s) for s in power_sums]
    sp = [conv(s) for s in splits] if plan.exact else [float(s) for s in splits]
    row = FirstOrderRow(lab, name, plan.voxels, plan.exact, plan.low, int(bin_width), plan.n_levels,
                        features(plan, hist, ps, band_count, conv(band_sum), sp, spacing, shift), hist,
                        dict(zip(PERCENTILES, plan.percentiles)), plan.base if plan.exact else plan.mean, ps,
                        int(band_count), conv(band_sum), sp)
    return row


def int_sums_from_words(words):
    """The five Python ints S1, S2, S3, S4, S_B of a row's ten uint64 words of lm_first_order_sums_dev."""
    w = [int(x) for x in np.asarray(words, dtype=np.uint64)]
    return [w[2 * k] | (w[2 * k + 1] << 64) for k in range(5)]

