"""First-order features on the host (no GPU): the feature code of lungmask_b200.first_order, fed by its numpy statement
of the two passes (sums_host), against the numpy statement of PyRadiomics' formulas in tests/_first_order_ref.py, and
the exact-sum identities against brute-force Fraction sums."""
import csv
import json
import math
from fractions import Fraction

import numpy as np
import pytest

from lungmask_b200 import first_order as fo

from _first_order_ref import first_order_ref

SPACING = (0.7, 0.8, 2.5)


def host_row(values, bw=25, shift=0, spacing=SPACING, label=1):
    """The FirstOrderRow of one ROI: the statistics as lm_label_stats_dev gives them (numpy.percentile of the float64
    values), the plan, sums_host, then build_row."""
    v = np.asarray(values).reshape(-1)
    x = v.astype(np.float64)
    plan = fo.plan_row(v.size, float(x.min()), float(x.max()), float(np.mean(x)), np.percentile(x, fo.PERCENTILES), bw,
                       v.dtype.kind in "iub")
    return fo.build_row(label, "roi", bw, plan, *fo.sums_host(v, plan, bw), spacing=spacing, shift=shift)


def check_against_ref(values, bw=25, shift=0, spacing=SPACING, exact=None):
    row = host_row(values, bw, shift, spacing)
    if exact is not None:
        assert row.exact is exact
    ref = first_order_ref(values, bw, shift, spacing)
    for k in fo.FIRST_ORDER_FEATURES:
        got, want = row.features[k], float(ref[k])
        if math.isnan(want):
            assert math.isnan(got), k
        elif k == "Skewness":
            assert abs(got - want) <= 1e-12 * (1 + abs(want)), (k, got, want)
        else:
            assert abs(got - want) <= 1e-12 * abs(want), (k, got, want)
    return row


def ct_values(rng, n, dtype):
    v = np.concatenate([rng.normal(-850, 60, n // 2), rng.normal(-300, 200, n - n // 2)])
    return np.clip(np.round(v), -1024, 3071).astype(dtype)


@pytest.mark.parametrize("dtype", [np.int16, np.int64, np.uint8, np.int8, np.int32])
def test_integer_rows_are_exact(dtype):
    rng = np.random.default_rng(1)
    if dtype in (np.uint8, np.int8):
        v = rng.integers(np.iinfo(dtype).min, np.iinfo(dtype).max, 5000, endpoint=True).astype(dtype)
        check_against_ref(v, bw=5, exact=True)
    else:
        check_against_ref(ct_values(rng, 20000, dtype), exact=True)


def test_int64_wide_range_takes_the_float_path():
    rng = np.random.default_rng(2)
    v = rng.integers(-10, 3000, 4000).astype(np.int64)
    v[0], v[1] = -(1 << 19), (1 << 19) + 5      # span 2^20 + 5
    check_against_ref(v, bw=5000, exact=False)
    edge = np.maximum(v, 0)
    edge[0], edge[1] = 0, (1 << 20) - 1          # span 2^20 - 1: still exact
    check_against_ref(edge, bw=5000, exact=True)
    edge[1] = 1 << 20                            # span 2^20: float
    check_against_ref(edge, bw=5000, exact=False)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_rows(dtype):
    rng = np.random.default_rng(3)
    v = (ct_values(rng, 20000, np.float64) + rng.random(20000)).astype(dtype)
    row = check_against_ref(v, exact=False)
    assert isinstance(row.power_sums[0], float)


def test_negative_values_and_bin_edges():
    v = np.array([-1000, -975, -976, -951, -950, -25, -26, 0, -1, 24, 25, 49, 50], np.int16)
    row = check_against_ref(v)
    assert row.low == -1000
    f = np.array([25.0, np.nextafter(25.0, -np.inf), 0.0, np.nextafter(0.0, -np.inf), -25.0, np.nextafter(-25.0, -np.inf),
                  50.0, 74.75], np.float64)
    row = check_against_ref(f)
    assert row.low == -50 and row.n_levels == 5
    assert list(row.histogram) == [1, 2, 2, 1, 2]


def test_constant_roi_and_single_voxel():
    for v in (np.full(37, -812, np.int16), np.full(11, -812.25, np.float32), np.array([7], np.int16),
              np.array([-3.5], np.float64)):
        row = check_against_ref(v)
        assert row.features["Skewness"] == 0.0 and row.features["Kurtosis"] == 0.0
        assert row.features["Variance"] == 0.0 and row.features["MeanAbsoluteDeviation"] == 0.0


def test_fractional_band_edges_with_ties():
    # n = 12: P10 at rank 1.1 and P90 at rank 9.9 fall between ties, so the band edges hold several equal values
    for v in (np.array([1, 2, 2, 2, 5, 5, 6, 9, 9, 9, 9, 12], np.int16),
              np.array([1, 2, 2, 2, 5, 5, 6, 9, 9, 9, 9, 12], np.float32) * np.float32(0.5),
              np.array([0, 10], np.int16)):                # no value inside [P10, P90] = [1, 9]
        row = check_against_ref(v)
    assert math.isnan(row.features["RobustMeanAbsoluteDeviation"]) and row.band_count == 0


@pytest.mark.parametrize("shift", [0, 1024, -2000, 7])
def test_shift(shift):
    rng = np.random.default_rng(4)
    check_against_ref(ct_values(rng, 3000, np.int16), shift=shift)
    check_against_ref(ct_values(rng, 3000, np.float32) + np.float32(0.25), shift=shift)


def test_no_spacing():
    row = check_against_ref(np.array([1, 2, 3], np.int16), spacing=None)
    assert math.isnan(row.features["TotalEnergy"])
    assert row.to_dict()["features"]["TotalEnergy"] is None


@pytest.mark.parametrize("seed", range(6))
def test_exact_identities_against_fractions(seed):
    """Moments, split-based mean absolute deviations and Energy of an exact row equal the brute-force Fraction values
    rounded once."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    v = rng.integers(-1024, 200, n).astype(np.int16)
    if seed == 5:
        v[:] = v[0]
    shift = int(rng.integers(-50, 50))
    row = host_row(v, shift=shift)
    assert row.exact
    xs = [int(a) for a in v]
    mu = Fraction(sum(xs), n)
    m = [sum((Fraction(a) - mu) ** k for a in xs) / n for k in (2, 3, 4)]
    f = row.features
    assert f["Variance"] == float(m[0])
    assert f["Kurtosis"] == (0.0 if m[0] == 0 else float(m[2] / m[0] ** 2))
    assert f["Mean"] == float(mu)
    assert f["MeanAbsoluteDeviation"] == float(sum(abs(Fraction(a) - mu) for a in xs) / n)
    e = sum((a + shift) ** 2 for a in xs)
    assert f["Energy"] == float(e)
    assert f["RootMeanSquared"] == math.sqrt(float(Fraction(e, n)))
    p10, p90 = np.percentile(v.astype(np.float64), [10, 90])
    band = [a for a in xs if p10 <= a <= p90]
    mb = Fraction(sum(band), len(band))
    assert f["RobustMeanAbsoluteDeviation"] == float(sum(abs(Fraction(a) - mb) for a in band) / len(band))
    # the power sums themselves
    d = [a - row.origin for a in xs]
    assert row.power_sums == [sum(x ** k for x in d) for k in (1, 2, 3, 4)]


def test_arguments():
    for bad in (1.5, True, "2", None):
        with pytest.raises(TypeError):
            fo.check_shift(bad)
    assert fo.check_shift(np.int16(-3)) == -3
    with pytest.raises(ValueError, match=r"first_order: row 3 \(x\) spans 257 grey levels"):
        fo.plan_row(10, -1024.0, 5375.0, 0.0, (0.0,) * 5, 25, True, "row 3 (x)")
    with pytest.raises(ValueError, match="first_order: row 1 .*non-finite"):
        fo.plan_row(10, -1.0, float("inf"), 0.0, (0.0,) * 5, 25, False, "row 1 (x)")


def test_writers(tmp_path):
    from lungmask_b200.io import save_first_order
    rows = [host_row(np.array([-900, -850, -851, -700], np.int16), label=1),
            fo.build_row(2, "absent", 25),
            host_row(np.array([-900.5, -12.25], np.float32), label=256)]
    res = fo.FirstOrderFeatures(SPACING, 25, 0, rows)
    save_first_order(str(tmp_path / "f.json"), res)
    d = json.loads((tmp_path / "f.json").read_text())
    assert d["bin_width"] == 25 and d["voxel_array_shift"] == 0 and len(d["rows"]) == 3
    assert d["rows"][0]["power_sums"] == rows[0].power_sums and d["rows"][0]["exact"] is True
    assert d["rows"][1]["features"]["Mean"] is None and d["rows"][2]["label"] == "lung"
    save_first_order(str(tmp_path / "f.csv"), res)
    lines = list(csv.reader((tmp_path / "f.csv").open()))
    assert lines[0] == list(fo.FirstOrderRow.SUMMARY) + list(fo.FIRST_ORDER_FEATURES)
    assert len(lines) == 4 and lines[2][4] == ""
    assert float(lines[1][lines[0].index("Mean")]) == rows[0].features["Mean"]
    with pytest.raises(SystemExit):
        save_first_order(str(tmp_path / "f.txt"), res)


def test_cli_flags(tmp_path):
    from lungmask_b200.__main__ import build_parser
    src = str(tmp_path / "in.npy")
    np.save(src, np.zeros((1, 2, 2), np.int16))
    a = build_parser().parse_args([src, "out.npy"])
    assert a.first_order is None and a.first_order_bin_width == 25 and a.first_order_shift == 0
    a = build_parser().parse_args([src, "out.npy", "--first-order", "f.csv", "--first-order-bin-width", "10",
                                   "--first-order-shift", "1024"])
    assert (a.first_order, a.first_order_bin_width, a.first_order_shift) == ("f.csv", 10, 1024)
