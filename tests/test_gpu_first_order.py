"""First-order features on the GPU (LMInferer.first_order, lm_first_order_sums_dev, lm_first_order_splits_dev) against
the host statements of lungmask_b200.first_order and tests/_first_order_ref.py: on exact rows the level histograms, the
power and split sums and the features are bit-identical to the host integer statement; float rows match the numpy
statement of PyRadiomics' formulas within the tolerances of the host tests."""
import json
import math

import numpy as np
import pytest

from lungmask_b200 import first_order as fo
from oracle import synth

from _first_order_ref import first_order_ref

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 2.5)   # (x, y, z) mm


@pytest.fixture(scope="module")
def inf():
    import os
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=47, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def two_lungs(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


def five_lobes(mask):
    S, H, _ = mask.shape
    z, y, _ = np.ogrid[:S, :H, :1]
    lobes = mask.copy()
    lobes[(mask == 1) & (z >= S // 2)] = 2
    lobes[(mask == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(mask == 2) & (z < S // 2)] = 4
    lobes[(mask == 2) & (z >= S // 2)] = 5
    return lobes


def random_labels(seed, shape, labels):
    import scipy.ndimage as ndi
    rng = np.random.default_rng(seed)
    field = ndi.gaussian_filter(rng.standard_normal(shape), 1.5)
    m = (field > np.quantile(field, 0.4)).astype(np.uint8)
    region = ndi.gaussian_filter(rng.standard_normal(shape), 2.5)
    cuts = np.quantile(region, np.linspace(0, 1, labels + 1)[1:-1])
    return m * (np.searchsorted(cuts, region) + 1).astype(np.uint8)


def rows_of(inf, mask):
    present = [int(x) for x in np.unique(mask) if x]
    return sorted(set(present) | set(range(1, inf.engine.n_classes[0]))) + [256]


def roi(vol, mask, r):
    v = vol[(mask > 0) if r == 256 else (mask == r)]
    return v[~np.isnan(v)] if v.dtype.kind == "f" else v


def host_expected(inf, vol, mask, bw=25, shift=0, spacing=SPACING):
    """The host rows: plan from the numpy statistics, sums_host, build_row (the names taken from the device rows)."""
    out = {}
    for r in rows_of(inf, mask):
        v = roi(vol, mask, r)
        if v.size == 0:
            out[r] = None
            continue
        x = v.astype(np.float64)
        plan = fo.plan_row(v.size, float(x.min()), float(x.max()), float(np.mean(x)), np.percentile(x, fo.PERCENTILES), bw,
                           vol.dtype.kind in "iub")
        out[r] = (plan, fo.sums_host(v, plan, bw))
    return out


def check_exact(inf, vol, mask, bw=25, shift=0, spacing=SPACING, expect_exact=None):
    res = inf.first_order(vol, mask, bin_width=bw, spacing=spacing, voxel_array_shift=shift)
    want = host_expected(inf, vol, mask, bw, shift, spacing)
    assert [r.label for r in res.rows] == [("lung" if r == 256 else r) for r in want]
    for row, (r, w) in zip(res.rows, want.items()):
        if w is None:
            assert row.voxels == 0 and all(math.isnan(v) for v in row.features.values()), r
            continue
        plan, sums = w
        if expect_exact is not None:
            assert row.exact is expect_exact.get(r, plan.exact), r
        if not plan.exact:
            check_float_row(row, roi(vol, mask, r), bw, shift, spacing)
            assert np.array_equal(row.histogram, sums[0]), r
            continue
        exp = fo.build_row(r, row.name, bw, plan, *sums, spacing=spacing, shift=shift)
        assert json.dumps(row.to_dict()) == json.dumps(exp.to_dict()), r
        assert all(a == b or (math.isnan(a) and math.isnan(b))
                   for a, b in zip(row.features.values(), exp.features.values())), r
    return res


def check_float_row(row, values, bw, shift, spacing):
    ref = first_order_ref(values, bw, shift, spacing)
    for k in fo.FIRST_ORDER_FEATURES:
        got, want = row.features[k], float(ref[k])
        if math.isnan(want):
            assert math.isnan(got), k
        elif k == "Skewness":
            assert abs(got - want) <= 1e-12 * (1 + abs(want)), (row.label, k, got, want)
        else:
            assert abs(got - want) <= 1e-12 * abs(want), (row.label, k, got, want)


def integer_volume(vol16, dtype):
    if dtype == np.uint8:
        return np.clip((vol16.astype(np.int32) + 1024) // 16, 0, 255).astype(np.uint8)
    if dtype == np.int8:
        return np.clip(vol16.astype(np.int32) // 16, -128, 127).astype(np.int8)
    return vol16.astype(dtype)


@pytest.mark.parametrize("dtype", [np.uint8, np.int8, np.int16, np.int32, np.int64])
@pytest.mark.parametrize("lobes", [False, True])
def test_integer_phantoms_bit_exact(inf, dtype, lobes):
    vol = integer_volume(synth.phantom(40, 96, 112, seed=5), dtype)
    mask = two_lungs(40, 96, 112)
    if lobes:
        mask = five_lobes(mask)
    check_exact(inf, vol, mask, bw=25 if vol.dtype.itemsize > 1 else 3, shift=7, expect_exact={})


def test_forty_labels_take_the_global_path(inf):
    mask = random_labels(9, (24, 40, 61), 40)
    assert len(np.unique(mask)) == 41
    vol = synth.phantom(24, 40, 61, seed=9)
    check_exact(inf, vol, mask)


def test_both_sides_of_the_exact_span(inf):
    """Label 1 spans less than 2^20 (exact), label 2 and the union more (float path)."""
    vol = synth.phantom(20, 64, 80, seed=6).astype(np.int32)
    mask = two_lungs(20, 64, 80)
    vol[mask == 2] *= 1000
    vmax = int(vol[mask > 0].max()) - int(vol[mask > 0].min())
    assert vmax >= fo.EXACT_SPAN and int(np.ptp(vol[mask == 1])) < fo.EXACT_SPAN
    res = check_exact(inf, vol, mask, bw=10000, expect_exact={1: True, 2: False, 256: False})
    assert isinstance(res["lung"].power_sums[0], float) and isinstance(res[1].power_sums[0], int)


def test_raw_sums_and_level_histograms(inf):
    """lm_first_order_sums_dev / lm_first_order_splits_dev against sums_host, and the histograms against np.bincount of
    lm_texture_levels_dev's map."""
    import torch
    vol = synth.phantom(30, 64, 72, seed=8)
    mask = five_lobes(two_lungs(30, 64, 72))
    tv, tm = _cuda(vol), _cuda(mask)
    res = inf.first_order(tv, tm)
    lev = torch.empty(vol.shape, dtype=torch.uint8, device="cuda:0")
    for row in res.rows:
        r = 256 if row.label == "lung" else row.label
        if not row.voxels:
            continue
        inf.engine.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), vol.shape, r, row.low, 25, row.n_levels, lev.data_ptr())
        L = lev.cpu().numpy()
        assert np.array_equal(row.histogram, np.bincount(L[L > 0], minlength=row.n_levels + 1)[1:]), r
        x = roi(vol, mask, r).astype(np.float64)
        plan = fo.plan_row(x.size, x.min(), x.max(), x.mean(), np.percentile(x, fo.PERCENTILES), 25, True)
        hist, S, nb, sb, splits = fo.sums_host(roi(vol, mask, r), plan, 25)
        assert row.power_sums == S and row.band_count == nb and row.band_sum == sb and row.splits == splits, r
        assert np.array_equal(row.histogram, hist), r


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "float32", "float64"])
def test_float_volumes_with_nan(inf, dtype):
    import torch
    rng = np.random.default_rng(11)
    base = synth.phantom(30, 64, 72, seed=11).astype(np.float64) + rng.random((30, 64, 72))
    base[rng.random(base.shape) < 0.02] = np.nan
    mask = five_lobes(two_lungs(30, 64, 72))
    t = torch.from_numpy(base).to(getattr(torch, dtype))
    values = t.float().numpy().astype(np.float64) if dtype in ("float16", "bfloat16") else t.numpy()
    res = inf.first_order(t.to("cuda:0"), _cuda(mask), spacing=SPACING, voxel_array_shift=1024)
    for row in res.rows:
        r = 256 if row.label == "lung" else row.label
        v = roi(values, mask, r)
        assert row.voxels == v.size and row.exact is False, r
        check_float_row(row, v, 25, 1024, SPACING)
        f = np.floor(v.astype(np.float64)).astype(np.int64)
        assert np.array_equal(row.histogram, np.bincount((f - row.low) // 25 + 1, minlength=row.n_levels + 1)[1:]), r


def test_cuda_tensor_and_numpy_agree(inf):
    vol = synth.phantom(20, 64, 72, seed=12)
    mask = five_lobes(two_lungs(20, 64, 72))
    a = inf.first_order(vol, mask, spacing=SPACING)
    tv, tm = _cuda(vol), _cuda(mask)
    b = inf.first_order(tv, tm, spacing=SPACING)
    assert json.dumps(a.to_dict()) == json.dumps(b.to_dict())
    assert np.array_equal(tv.cpu().numpy(), vol) and np.array_equal(tm.cpu().numpy(), mask)


def test_absent_model_labels(inf):
    vol = synth.phantom(10, 32, 40, seed=13)
    mask = (two_lungs(10, 32, 40) == 2).astype(np.uint8) * 2
    res = inf.first_order(vol, mask)
    assert res[1].voxels == 0 and res[1].exact is None
    assert all(math.isnan(v) for v in res[1].features.values())
    assert res[2].voxels == res["lung"].voxels > 0


def test_refusals_before_any_kernel(inf, monkeypatch):
    from lungmask_b200 import _native
    vol = synth.phantom(10, 32, 40, seed=14).astype(np.float32)
    mask = two_lungs(10, 32, 40)

    def no_kernel(*a, **k):
        raise AssertionError("a first-order kernel ran")
    monkeypatch.setattr(inf.engine, "first_order_sums_dev", no_kernel)
    monkeypatch.setattr(inf.engine, "first_order_splits_dev", no_kernel)
    for v in (np.inf, -np.inf):
        bad = vol.copy()
        bad[mask == 1] = np.where(np.arange((mask == 1).sum()) == 3, v, bad[mask == 1])
        with pytest.raises(ValueError, match="non-finite"):
            inf.first_order(bad, mask)
    wide = vol.copy()
    wide[mask == 2] *= 10
    with pytest.raises(ValueError, match="first_order: row .* grey levels"):
        inf.first_order(wide, mask, bin_width=1)
    with pytest.raises(TypeError):
        inf.first_order(vol, mask, voxel_array_shift=0.5)
    with pytest.raises(ValueError):
        inf.first_order(vol, mask, bin_width=0)
    with pytest.raises(TypeError):
        inf.first_order(vol, mask, bin_width=2.5)
    monkeypatch.undo()
    # the C entry points check their row arguments
    tv, tm = _cuda(vol), _cuda(mask)
    z = np.zeros(257)
    mode = np.zeros(257, np.int32)
    mode[1] = fo.MODE_FLOAT
    with pytest.raises(_native.NativeError, match="union row"):
        inf.engine.first_order_sums_dev(tv.data_ptr(), _native.DTYPE_F32, tm.data_ptr(), vol.shape, 25, mode, z,
                                        np.ones(257), z, z, z, z)
    mode[256] = fo.MODE_EXACT
    with pytest.raises(_native.NativeError, match="integer volume"):
        inf.engine.first_order_sums_dev(tv.data_ptr(), _native.DTYPE_F32, tm.data_ptr(), vol.shape, 25, mode, z,
                                        np.ones(257), z, z, z, z)


def test_full_size_int16_bit_exact(inf):
    vol = synth.phantom(300, 512, 512, seed=100)
    mask = two_lungs(300, 512, 512)
    res = check_exact(inf, vol, mask)
    assert all(r.exact for r in res.rows if r.voxels)


def test_cli_writes_json_and_csv(tmp_path):
    import csv
    import torch
    from lungmask_b200.__main__ import main
    p = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.npy")
    np.save(src, synth.phantom(6, 96, 96, seed=21))
    js, cs = str(tmp_path / "fo.json"), str(tmp_path / "fo.csv")
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--first-order", js, "--first-order-shift", "1024"])
    main([src, str(tmp_path / "m2.npy"), "--modelpath", p, "--noprogress", "--first-order", cs, "--first-order-bin-width", "10"])
    d = json.loads(open(js).read())
    assert d["voxel_array_shift"] == 1024 and d["bin_width"] == 25 and d["rows"][-1]["label"] == "lung"
    lines = list(csv.reader(open(cs)))
    assert lines[0] == list(fo.FirstOrderRow.SUMMARY) + list(fo.FIRST_ORDER_FEATURES)
    assert all(l[5] == "10" for l in lines[1:])
