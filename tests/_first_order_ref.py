"""A numpy statement of PyRadiomics' default firstorder features, written from the published formulas (PyRadiomics
documentation, "First Order Features"), for the ROI values of one row: no resampling, no resegmentation, fixed bin width.

The values are taken as float64.  Mean, Variance (population), Skewness m3 / m2^1.5 and Kurtosis m4 / m2^2 (both 0 when
m2 = 0) come from the deviations about numpy's mean; the percentiles from numpy.percentile, Median from numpy.median;
RobustMeanAbsoluteDeviation over P10 <= x <= P90; Entropy and Uniformity from the histogram of the levels
floor((floor(x) - low) / bw) + 1, low = bw * floor(min / bw)."""
import math

import numpy as np

EPS = np.spacing(1)


def first_order_ref(values, bin_width=25, shift=0, spacing=None):
    x = np.asarray(values).reshape(-1).astype(np.float64)
    n = x.size
    p10, p25, p75, p90 = np.percentile(x, [10, 25, 75, 90])
    mean = np.mean(x)
    dev = x - mean
    m2, m3, m4 = np.mean(dev ** 2), np.mean(dev ** 3), np.mean(dev ** 4)
    band = x[(x >= p10) & (x <= p90)]
    energy = np.sum((x + shift) ** 2)
    f = np.floor(x)
    low = bin_width * math.floor(f.min() / bin_width)
    levels = ((f - low) // bin_width + 1).astype(np.int64)
    p = np.bincount(levels)[1:] / n
    return {
        "10Percentile": p10,
        "90Percentile": p90,
        "Energy": energy,
        "Entropy": -np.sum(p * np.log2(p + EPS)),
        "InterquartileRange": p75 - p25,
        "Kurtosis": 0.0 if m2 == 0 else m4 / m2 ** 2,
        "Maximum": np.max(x),
        "MeanAbsoluteDeviation": np.mean(np.abs(dev)),
        "Mean": mean,
        "Median": np.median(x),
        "Minimum": np.min(x),
        "Range": np.max(x) - np.min(x),
        "RobustMeanAbsoluteDeviation": np.mean(np.abs(band - band.mean())) if band.size else float("nan"),
        "RootMeanSquared": math.sqrt(energy / n),
        "Skewness": 0.0 if m2 == 0 else m3 / m2 ** 1.5,
        "TotalEnergy": float(np.prod(spacing)) * energy if spacing is not None else float("nan"),
        "Uniformity": np.sum(p ** 2),
        "Variance": m2,
    }
