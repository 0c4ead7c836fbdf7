"""The numpy statement of the voxel-based first-order maps (first_order_maps.maps_host) against a literal per-voxel loop
over first_order.sums_host / features and tests/_first_order_ref.py, and the argument checks (CPU only)."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from _first_order_ref import first_order_ref  # noqa: E402

from lungmask_b200 import first_order as fo  # noqa: E402
from lungmask_b200 import first_order_maps as fm  # noqa: E402

ORDER_STATS = ("10Percentile", "90Percentile", "Median", "InterquartileRange", "Minimum", "Maximum", "Range")


def literal_maps(vol, mask, label, r, masked, bw, shift, spacing):
    """Per ROI voxel: the window's candidate values through first_order.sums_host + features (order statistics from
    numpy.percentile), in a plain loop."""
    roi = fm.roi_of(vol, mask, label)
    x = np.asarray(vol)
    if x.dtype == np.float16:
        x = x.astype(np.float32)
    cand = roi if masked else (~np.isnan(x) if x.dtype.kind == "f" else np.ones(x.shape, bool))
    integer = x.dtype.kind in "iub"
    out = {}
    for c in zip(*np.nonzero(roi)):
        sl = tuple(slice(max(c[k] - r, 0), c[k] + r + 1) for k in range(3))
        v = x[sl][cand[sl]]
        xv = v.astype(np.float64)
        pc = np.percentile(xv, fo.PERCENTILES)
        plan = fo.plan_row(v.size, float(xv.min()), float(xv.max()), float(xv.mean()), pc, bw, integer)
        f = fo.features(plan, *fo.sums_host(v, plan, bw), spacing=spacing, shift=shift)
        ref = first_order_ref(v, bw, shift, spacing)
        for k in ORDER_STATS:
            f[k] = float(ref[k])
        out[c] = f
    return out


def assert_maps_match(res, lit, feats=fo.FIRST_ORDER_FEATURES):
    for c, f in lit.items():
        for k in feats:
            got, want = res.maps[k][c], f[k]
            if k in ORDER_STATS:
                assert got == want, (c, k, got, want)
            elif math.isnan(want):
                assert math.isnan(got), (c, k, got)
            else:
                assert abs(got - want) <= 1e-12 * max(abs(want), 1.0), (c, k, got, want)


def volume(kind, shape, rng):
    if kind == "int16":
        return rng.integers(-1000, 200, shape).astype(np.int16)
    if kind == "int32wide":
        return rng.integers(-(1 << 22), 1 << 22, shape).astype(np.int32)
    v = (rng.normal(-600, 200, shape)).astype(np.float32)
    v[rng.random(shape) < 0.1] = np.nan
    return v


@pytest.mark.parametrize("kind", ["int16", "int32wide", "float32"])
@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("masked", [True, False])
def test_maps_host_against_loop(kind, r, masked):
    rng = np.random.default_rng(7 * r + (kind == "float32") + 3 * masked)
    shape = (5, 6, 7)
    vol = volume(kind, shape, rng)
    mask = rng.integers(0, 3, shape).astype(np.uint8)
    bw = 25 if kind != "int32wide" else 1 << 16
    res = fm.maps_host(vol, mask, "lung", kernel_radius=r, masked_kernel=masked, bin_width=bw, voxel_array_shift=7,
                       spacing=(0.7, 0.8, 1.5))
    assert res.exact == (kind == "int16")
    assert_maps_match(res, literal_maps(vol, mask, "lung", r, masked, bw, 7, (0.7, 0.8, 1.5)))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 2, 1), (2, 1, 2), (1, 4, 3), (3, 1, 1)])
@pytest.mark.parametrize("init", [0.0, float("nan")])
def test_small_extents_label_row_and_init_value(shape, init):
    rng = np.random.default_rng(11)
    vol = rng.integers(-1000, 100, shape).astype(np.int16)
    mask = rng.integers(0, 3, shape).astype(np.uint8)
    mask.reshape(-1)[0] = 2
    res = fm.maps_host(vol, mask, 2, kernel_radius=2, init_value=init)
    assert res.spacing is None and np.isnan(res["TotalEnergy"][mask == 2]).all()
    assert_maps_match(res, literal_maps(vol, mask, 2, 2, True, 25, 0, None))
    outside = mask != 2
    for k, m in res.maps.items():
        assert m.shape == shape and m.dtype == np.float64
        if math.isnan(init):
            assert np.isnan(m[outside]).all()
        else:
            assert (m[outside] == init).all()


def test_windows_clipped_by_every_face_and_nan_under_mask():
    rng = np.random.default_rng(3)
    vol = rng.normal(0, 50, (4, 5, 6)).astype(np.float32)
    vol[0, 0, 0] = np.nan
    vol[3, 4, 5] = np.nan
    mask = np.ones(vol.shape, np.uint8)
    res = fm.maps_host(vol, mask, kernel_radius=1, masked_kernel=False, init_value=-5.0)
    assert res.voxels == vol.size - 2
    assert res["Mean"][0, 0, 0] == -5.0 and res["Mean"][3, 4, 5] == -5.0
    assert_maps_match(res, literal_maps(vol, mask, "lung", 1, False, 25, 0, None))


def test_one_voxel_roi():
    vol = np.arange(27, dtype=np.int16).reshape(3, 3, 3) - 500
    mask = np.zeros(vol.shape, np.uint8)
    mask[1, 1, 1] = 1
    res = fm.maps_host(vol, mask)
    c = (1, 1, 1)
    for k in ("Variance", "Skewness", "Kurtosis", "MeanAbsoluteDeviation", "RobustMeanAbsoluteDeviation"):
        assert res[k][c] == 0.0, k
    assert res["Mean"][c] == res["Minimum"][c] == res["Maximum"][c] == float(vol[c])


def test_feature_subset_equals_full_planes():
    rng = np.random.default_rng(5)
    vol = rng.integers(-900, -100, (4, 6, 6)).astype(np.int16)
    mask = rng.integers(0, 2, vol.shape).astype(np.uint8)
    full = fm.maps_host(vol, mask, kernel_radius=2)
    sub = fm.maps_host(vol, mask, kernel_radius=2, features=("Entropy", "Mean", "Variance"))
    assert list(sub.maps) == ["Entropy", "Mean", "Variance"]
    for k, m in sub.maps.items():
        assert np.array_equal(m.view(np.uint64), full[k].view(np.uint64))


@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("kind", ["int16", "float32"])
def test_cover_case_equals_aggregate_features(r, kind):
    """A ROI inside an (r+1)^3 cube: any two of its voxels are at most r apart along every axis, so every ROI voxel's
    window holds the whole ROI and every map value is the aggregate first-order feature of the ROI."""
    rng = np.random.default_rng(r)
    shape = (2 * r + 3,) * 3
    vol = volume(kind, shape, rng)
    if kind == "float32":
        vol[np.isnan(vol)] = 1.0
    mask = np.zeros(shape, np.uint8)
    box = (slice(1, r + 2),) * 3
    mask[box] = (rng.random((r + 1,) * 3) < 0.6).astype(np.uint8)
    mask[1, 1, 1] = mask[r + 1, r + 1, r + 1] = 1
    res = fm.maps_host(vol, mask, kernel_radius=r, spacing=(1.0, 2.0, 0.5), voxel_array_shift=3)
    v = vol[mask > 0]
    xv = v.astype(np.float64)
    plan = fo.plan_row(v.size, float(xv.min()), float(xv.max()), float(xv.mean()), np.percentile(xv, fo.PERCENTILES), 25,
                       kind == "int16")
    agg = fo.features(plan, *fo.sums_host(v, plan, 25), spacing=(1.0, 2.0, 0.5), shift=3)
    for k in fo.FIRST_ORDER_FEATURES:
        got = res[k][mask > 0]
        if k in ("10Percentile", "90Percentile", "Median", "InterquartileRange", "Minimum", "Maximum", "Range"):
            assert (got == agg[k]).all(), k
        else:
            assert np.allclose(got, agg[k], rtol=1e-12, atol=1e-12), (k, got[:3], agg[k])


@pytest.mark.parametrize("v", [0, 1, -1, (1 << 53) - 1, 1 << 53, (1 << 53) + 1, (1 << 54) + 2, (1 << 54) + 6,
                               (1 << 64) - 1, 1 << 64, (1 << 64) + 1, (1 << 65) + (1 << 12), (1 << 65) + (1 << 12) + 1,
                               (1 << 117) - 1, -(1 << 100) - (1 << 47), -(1 << 100) - (1 << 47) - 1, (1 << 126) + 12345])
def test_int_to_float_matches_python(v):
    assert fm.int_to_float(v) == float(v)
    assert fm.int_to_float(v) == float(np.array([v], dtype=object).astype(np.float64)[0])


def test_int_to_float_random():
    rng = np.random.default_rng(1)
    for _ in range(2000):
        v = int(rng.integers(0, 1 << 62)) << int(rng.integers(0, 64)) | int(rng.integers(0, 1 << 62))
        v = -v if rng.random() < 0.5 else v
        assert fm.int_to_float(v) == float(v)


def test_entropy_table():
    T = fm.entropy_table(27)
    assert T.size == 27 * 28 // 2
    for N in (1, 5, 27):
        for h in (1, N):
            p = np.float64(h) / N
            assert T[N * (N - 1) // 2 + h - 1] == -(p * np.log2(p + np.spacing(1)))
    assert fm.entropy_table(343).size == 58996


def test_refusals():
    vol = np.zeros((3, 3, 3), np.int16)
    mask = np.ones((3, 3, 3), np.uint8)
    for r in (0, 4, 1.0, True):
        with pytest.raises(ValueError, match="kernel_radius"):
            fm.maps_host(vol, mask, kernel_radius=r)
    f = vol.astype(np.float32)
    f[1, 1, 1] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        fm.maps_host(f, mask)
    wide = np.arange(27, dtype=np.int16).reshape(3, 3, 3) * 100
    with pytest.raises(ValueError, match="bin width"):
        fm.maps_host(wide, mask, bin_width=1)
    with pytest.raises(ValueError, match="unknown first-order feature"):
        fm.maps_host(vol, mask, features=("Mean", "Mode"))
    with pytest.raises(TypeError):
        fm.maps_host(vol, mask, features="Mean")
    with pytest.raises(ValueError, match="empty"):
        fm.maps_host(vol, mask, features=())
    for lab in (0, 256, "left", -1):
        with pytest.raises(ValueError, match="label"):
            fm.maps_host(vol, mask, label=lab)
    with pytest.raises(ValueError):
        fm.maps_host(vol, mask, bin_width=0)
    with pytest.raises(ValueError, match="2\\^58"):
        fm.maps_host(vol, mask, voxel_array_shift=1 << 58)
    with pytest.raises(TypeError):
        fm.maps_host(vol, mask, voxel_array_shift=0.5)


def test_unmasked_region_is_padded_box():
    vol = np.zeros((7, 7, 7), np.int16)
    vol[0, 0, 0] = -3000      # outside the padded box: no effect on the levels
    vol[2, 3, 3] = -100
    mask = np.zeros(vol.shape, np.uint8)
    mask[3, 3, 3] = 1
    res = fm.maps_host(vol, mask, masked_kernel=False, bin_width=25)
    assert res.low == -100 and res.n_levels == 5
    vol[1, 3, 3] = -7000      # inside the box padded by 2: the r = 2 region sees it
    res2 = fm.maps_host(vol, mask, masked_kernel=False, kernel_radius=2, bin_width=100)
    assert res2.low == -7000


def test_empty_roi_holds_init_value():
    vol = np.zeros((2, 3, 4), np.float32)
    res = fm.maps_host(vol, np.zeros(vol.shape, np.uint8), init_value=float("nan"))
    assert res.voxels == 0 and res.low is None
    assert all(np.isnan(m).all() for m in res.maps.values())


def test_save_feature_maps_round_trip(tmp_path):
    from lungmask_b200.io import Volume, load_input_image, save_feature_maps
    rng = np.random.default_rng(2)
    vol = rng.integers(-1000, 0, (3, 5, 6)).astype(np.int16)
    mask = rng.integers(0, 2, vol.shape).astype(np.uint8)
    res = fm.maps_host(vol, mask, features=("Mean", "Entropy"), init_value=float("nan"))
    like = Volume(vol, (0.7, 0.8, 2.0), (1.0, -2.0, 3.0))
    for fmt in ("nii.gz", "nii", "mha", "npy"):
        paths = save_feature_maps(str(tmp_path / fmt), res, like, fmt)
        assert [os.path.basename(p) for p in paths] == ["lung_Entropy.%s" % fmt, "lung_Mean.%s" % fmt]
        for p, k in zip(paths, ("Entropy", "Mean")):
            img = load_input_image(p)
            assert np.array_equal(np.asarray(img.array).view(np.uint64), res[k].view(np.uint64))
            if fmt != "npy":
                assert np.allclose(img.spacing, like.spacing)
    with pytest.raises(ValueError, match="format"):
        save_feature_maps(str(tmp_path / "x"), res, like, "png")


def test_cli_flags_checked_before_segmentation(tmp_path):
    from lungmask_b200.__main__ import main
    src = str(tmp_path / "vol.npy")
    np.save(src, np.zeros((2, 4, 4), np.int16))
    f = tmp_path / "file"
    f.write_text("x")
    base = [src, str(tmp_path / "m.npy"), "--first-order-maps", str(tmp_path / "maps")]
    for extra, msg in ((["--first-order-maps-label", "0"], "--first-order-maps-label"),
                       (["--first-order-maps-label", "left"], "--first-order-maps-label"),
                       (["--first-order-maps-features", "Mean,Mode"], "--first-order-maps-features"),
                       (["--first-order-bin-width", "0"], "--first-order-bin-width")):
        with pytest.raises(SystemExit, match=msg):
            main(base + extra)
    with pytest.raises(SystemExit, match="not a directory"):
        main([src, str(tmp_path / "m.npy"), "--first-order-maps", str(f)])
    with pytest.raises(SystemExit, match="parent directory"):
        main([src, str(tmp_path / "m.npy"), "--first-order-maps", str(tmp_path / "no" / "maps")])
    for extra in (["--first-order-maps-radius", "4"], ["--first-order-maps-format", "png"]):
        with pytest.raises(SystemExit):
            main(base + extra)
