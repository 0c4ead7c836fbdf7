"""Regional statistics on the GPU (LMInferer.surface_distance / regional_statistics, lm_plane_label_counts_dev,
lm_surface_distance_dev, lm_region_map_dev): the distance transform against scipy.ndimage.distance_transform_edt, the
plane counts against np.bincount, and every zone / shell row against the numpy oracle of test_gpu_statistics applied to
the voxels the oracle's own zones and scipy's depths select."""
import json

import numpy as np
import pytest
from scipy import ndimage

from oracle import synth
from test_gpu_statistics import check, oracle

pytestmark = pytest.mark.gpu


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    import torch
    d = tmp_path_factory.mktemp("region_weights")
    paths = {}
    for K in (3, 6):
        paths[K] = str(d / ("w%d.pth" % K))
        torch.save(synth.random_state_dict(K, seed=60 + K, head_gain=0.3), paths[K])
    return paths


@pytest.fixture(scope="module")
def inf(weights):
    from lungmask_b200 import LMInferer
    return LMInferer(modelpath=weights[3], batch_size=4, tqdm_disable=True)


@pytest.fixture(scope="module")
def inf6(weights):
    from lungmask_b200 import LMInferer
    return LMInferer(modelpath=weights[6], batch_size=4, tqdm_disable=True)


def two_lungs(shape, seed=0):
    """int16 phantom and a two-lung uint8 mask: two ellipsoids, label 1 right (low x), 2 left, cut by the first slice."""
    n0, n1, n2 = shape
    vol = synth.phantom(n0, n1, n2, seed=seed)
    z, y, x = np.ogrid[:n0, :n1, :n2]
    mask = np.zeros(shape, np.uint8)
    for l, cx in ((1, 0.3), (2, 0.7)):
        e = ((z - 0.45 * n0) / (0.55 * n0)) ** 2 + ((y - 0.5 * n1) / (0.32 * n1)) ** 2 + ((x - cx * n2) / (0.17 * n2)) ** 2
        mask[e <= 1.0] = l
    return vol, mask


def scipy_depth(mask, spacing):
    return np.float32(ndimage.distance_transform_edt(mask > 0, sampling=spacing))


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    same_inf = np.isinf(a) & (a == b)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return np.where(same_inf, 0, np.abs(ia - ib))


def compare_edt(inf, mask, spacing, exact):
    got = inf.surface_distance(mask, spacing)
    assert got.dtype == np.float32 and got.shape == mask.shape
    tm = _cuda(mask)
    before = tm.clone()
    got_t = inf.surface_distance(tm, spacing)
    assert got_t.is_cuda and got_t.dtype.is_floating_point and np.array_equal(got_t.cpu().numpy(), got)
    assert bool((tm == before).all()), "the mask tensor was modified"
    if (mask > 0).all():
        assert np.isposinf(got).all()
        return
    want = scipy_depth(mask, spacing)
    if exact:
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), float(np.abs(got - want).max())
    else:
        assert _ulps(got, want).max() <= 1


EXACT = [(1.0, 1.0, 1.0), (2.5, 0.703125, 0.703125), (0.625, 0.75, 1.25)]


def _blobs(shape, seed):
    rng = np.random.default_rng(seed)
    m = ndimage.gaussian_filter(rng.random(shape), 1.5) > 0.48
    return (m * rng.integers(1, 4, shape)).astype(np.uint8)


@pytest.mark.parametrize("spacing", EXACT)
def test_edt_exact_odd_shapes(inf, spacing):
    for shape, seed in (((37, 45, 53), 1), ((1, 61, 47), 2), ((2, 33, 71), 3), ((5, 1, 9), 4), ((3, 7, 1), 5)):
        compare_edt(inf, _blobs(shape, seed), spacing, exact=True)


def test_edt_within_one_ulp(inf):
    compare_edt(inf, _blobs((37, 45, 53), 6), (1.25, 0.7, 0.7), exact=False)
    _, m = two_lungs((24, 96, 112), seed=2)
    compare_edt(inf, m, (1.25, 0.7, 0.7), exact=False)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_edt_long_lines(inf, axis):
    shape = [3, 5, 6]
    shape[axis] = 1300
    rng = np.random.default_rng(10 + axis)
    m = (rng.random(shape) > 0.004).astype(np.uint8)
    m[1, 2, 3] = 1
    compare_edt(inf, m, (2.5, 0.703125, 0.625), exact=True)
    line = np.ones(shape, np.uint8)                      # one background voxel on the whole long line
    idx = [1, 2, 3]
    idx[axis] = 700
    line[tuple(idx)] = 0
    compare_edt(inf, line, (1.0, 1.0, 1.0), exact=True)


def test_edt_special_masks(inf):
    m = np.ones((9, 11, 13), np.uint8) * 2
    m[4, 5, 6] = 0                                       # a single background voxel
    compare_edt(inf, m, (2.5, 0.703125, 0.703125), exact=True)
    compare_edt(inf, np.zeros((9, 11, 13), np.uint8), (1.0, 1.0, 1.0), exact=True)
    assert (inf.surface_distance(np.zeros((9, 11, 13), np.uint8), (1, 1, 1)) == 0).all()
    full = np.ones((9, 11, 13), bool)
    compare_edt(inf, full, (1.0, 1.0, 1.0), exact=True)   # no zero voxel: +inf everywhere (scipy differs here)
    import torch
    cpu = inf.surface_distance(torch.from_numpy(m), (1.0, 1.0, 1.0))
    assert isinstance(cpu, torch.Tensor) and not cpu.is_cuda


def test_edt_two_lung_phantom(inf):
    _, m = two_lungs((96, 512, 512), seed=3)
    compare_edt(inf, m, (2.5, 0.703125, 0.703125), exact=True)


def test_plane_counts(inf6):
    eng = inf6.engine
    rng = np.random.default_rng(12)
    m = _blobs((23, 41, 37), 7) * rng.integers(1, 90, (23, 41, 37)).astype(np.uint8)
    m[0, 0, 0] = 255
    tm = _cuda(m)
    for axis in range(3):
        got = eng.plane_label_counts_dev(tm.data_ptr(), m.shape, axis)
        moved = np.moveaxis(m, axis, 0).reshape(m.shape[axis], -1)
        want = np.stack([np.bincount(p, minlength=256) for p in moved])
        assert np.array_equal(got[:, :256], want)
        assert np.array_equal(got[:, 256], (moved > 0).sum(axis=1))


# ---- the statistics oracle ----------------------------------------------------------------------------------------------
def oracle_zones(sel, axis, superior_high, zones, zone_by):
    """The zone of every plane of a row, a direct loop statement of the formulas (-1 outside the row)."""
    c = [int(x) for x in np.moveaxis(sel, axis, 0).reshape(sel.shape[axis], -1).sum(axis=1)]
    order = list(range(len(c)))[::-1] if superior_high else list(range(len(c)))
    occupied = [k for k, p in enumerate(order) if c[p]]
    out = [-1] * len(c)
    if not occupied:
        return np.array(out)
    a, b = occupied[0], occupied[-1]
    total = sum(c)
    before = 0
    for i in range(a, b + 1):
        ci = c[order[i]]
        if zone_by == "height":
            out[order[i]] = (zones * (i - a)) // (b - a + 1)
        else:
            out[order[i]] = min(zones - 1, (zones * (2 * before + ci)) // (2 * total))
        before += ci
    return np.array(out)


def check_regions(got, vol, mask, spacing_axes, axis, superior_high, zones, zone_by, shells, q, t):
    depth = scipy_depth(mask, spacing_axes) if shells else None
    labels = sorted(set(int(x) for x in np.unique(mask) if x))
    for l in labels + ["lung"]:
        sel = mask > 0 if l == "lung" else mask == l
        z = oracle_zones(sel, axis, superior_high, zones, zone_by)
        shape = [1, 1, 1]
        shape[axis] = -1
        plane_zone = z.reshape(shape)
        assert np.array_equal(got.profile[l], np.moveaxis(sel, axis, 0).reshape(sel.shape[axis], -1).sum(axis=1))
        for k in range(zones):
            part = (sel & (plane_zone == k)).astype(np.uint8)
            row = got.row(l, "zone", k)
            if part.any():
                check({1: row.stats}, {1: oracle(vol, part, q, t)[1]})
            else:
                assert row.stats.voxels == 0
            p = np.flatnonzero(z == k)
            assert row.planes == ((int(p[0]), int(p[-1])) if p.size else None)
        if shells:
            edges = [0.0] + list(shells) + [np.inf]
            for j in range(len(shells) + 1):
                part = (sel & (depth >= np.float32(edges[j])) & (depth < np.float32(edges[j + 1]))).astype(np.uint8)
                row = got.row(l, "shell", j)
                if part.any():
                    check({1: row.stats}, {1: oracle(vol, part, q, t)[1]})
                else:
                    assert row.stats.voxels == 0


Q, T = (15.0, 50.0), (-950, -910)


@pytest.mark.parametrize("zone_by", ["volume", "height"])
def test_statistics_against_oracle(inf6, zone_by):
    vol, mask = two_lungs((48, 160, 176), seed=5)
    mask[20:30][mask[20:30] == 1] = 3                    # a label with empty planes in its range: two slabs
    mask[24:26][mask[24:26] == 3] = 1
    mask[7, 80, 50] = 4                                  # a label on a single plane
    sp = (0.703125, 0.703125, 2.5)
    for zones in (1, 2, 3, 5):
        got = inf6.regional_statistics(vol, mask, spacing=sp, zones=zones, zone_by=zone_by, shells_mm=(5.0, 12.5),
                                       percentiles=Q, thresholds=T)
        check_regions(got, vol, mask, sp[::-1], 0, True, zones, zone_by, (5.0, 12.5), Q, T)
    assert [r.region_name for r in got.rows[:5]] == ["zone %d of 5" % k for k in range(1, 6)]
    # absent model label 5: zero voxels and NaN values in every row
    assert all(r.stats.voxels == 0 and np.isnan(r.stats.mean_hu) for r in got.rows if r.label == 5)
    assert sorted(set(r.label for r in got.rows), key=str) == sorted([1, 2, 3, 4, 5, "lung"], key=str)


def test_float_volume_and_tensors(inf6):
    import torch
    vol, mask = two_lungs((40, 128, 144), seed=6)
    rng = np.random.default_rng(3)
    vf = (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(np.float32)
    vf[rng.random(vol.shape) < 0.01] = np.nan
    sp = (0.75, 0.625, 1.25)
    a = inf6.regional_statistics(vf, mask, spacing=sp, percentiles=Q, thresholds=T)
    check_regions(a, vf, mask, sp[::-1], 0, True, 3, "volume", (10.0,), Q, T)
    assert [r.region_name for r in a.rows[:4]] == ["upper", "middle", "lower", "depth 0-10 mm"]
    tv, tm = _cuda(vf), _cuda(mask)
    bv, bm = tv.clone(), tm.clone()
    b = inf6.regional_statistics(tv, tm, spacing=sp, percentiles=Q, thresholds=T)
    assert torch.equal(tm, bm) and np.array_equal(tv.cpu().numpy().view(np.int32), bv.cpu().numpy().view(np.int32))
    da, db = a.to_dict(), b.to_dict()
    for ra, rb in zip(da["rows"], db["rows"]):
        for k in ("mean_hu", "std_hu"):
            x, y = ra["statistics"][k], rb["statistics"][k]
            if x is not None and y is not None and abs(x - y) <= 1e-12 * max(abs(x), 1.0):
                rb["statistics"][k] = x
    assert json.dumps(da) == json.dumps(db)


def test_stream_ordering(inf6):
    import torch
    vol, mask = two_lungs((32, 128, 128), seed=7)
    sp = (0.7, 0.7, 1.25)
    want = json.dumps(inf6.regional_statistics(vol, mask, spacing=sp).to_dict())
    src, srcm = _cuda(vol), _cuda(mask)
    side = torch.cuda.Stream(device=0)
    for use_side in (True, False):
        t = torch.full(vol.shape, -1000, dtype=torch.int16, device="cuda:0")
        tm = torch.zeros(mask.shape, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        with torch.cuda.stream(side if use_side else torch.cuda.default_stream(0)):
            torch.cuda._sleep(100_000_000)
            t.copy_(src)
            tm.copy_(srcm)
            got = inf6.regional_statistics(t, tm, spacing=sp)
            d = inf6.surface_distance(tm, sp[::-1])
        assert json.dumps(got.to_dict()) == want, "side stream" if use_side else "default stream"
        torch.cuda.synchronize()
        assert np.array_equal(d.cpu().numpy(), inf6.surface_distance(mask, sp[::-1]))


def _direction(code):
    d = np.zeros((3, 3))
    for c, ch in enumerate(code):
        r = "LPS".index(ch) if ch in "LPS" else "RAI".index(ch)
        d[r, c] = 1.0 if ch in "LPS" else -1.0
    return tuple(d.reshape(-1))


def test_orientations(inf6):
    from lungmask_b200 import io as lio, orient, regions as rg
    vol, mask = two_lungs((36, 112, 128), seed=8)
    sp = (0.703125, 0.625, 2.5)                            # LPS (x, y, z)
    want = inf6.regional_statistics(vol, mask, spacing=sp, zones=4, shells_mm=(4.0,))
    for code, axis, high in (("RAS", 0, True), ("PLI", 0, False), ("LIP", 1, False), ("SAL", 2, True)):
        assert rg.craniocaudal_axis(code) == (axis, high)
        phys = ["LPS".index(ch) if ch in "LPS" else "RAI".index(ch) for ch in code]
        v = lio.Volume(orient.from_lps(vol, code), tuple(sp[p] for p in phys), (0.0, 0.0, 0.0), _direction(code))
        got = inf6.regional_statistics(v, orient.from_lps(mask, code), zones=4, shells_mm=(4.0,))
        assert got.zone_axis == axis and got.superior_high == high
        assert [(r.label, r.region, r.index, r.region_name) for r in got.rows] == \
            [(r.label, r.region, r.index, r.region_name) for r in want.rows]
        for g, w in zip(got.rows, want.rows):
            assert json.dumps(g.stats.to_dict()) == json.dumps(w.stats.to_dict()), (code, g.label, g.region, g.index)
            assert (g.planes is None) == (w.planes is None)
            if g.planes is not None:
                assert g.planes[1] - g.planes[0] == w.planes[1] - w.planes[0]
        for l in want.profile:
            p = got.profile[l] if high else got.profile[l][::-1]
            assert np.array_equal(p, want.profile[l])


def test_errors(inf6):
    import torch
    from lungmask_b200 import _native
    vol, mask = two_lungs((16, 64, 64), seed=9)
    tv, tm = _cuda(vol), _cuda(mask)
    with pytest.raises(ValueError, match="spacing=.*shells_mm=\\(\\)"):
        inf6.regional_statistics(vol, mask)
    assert inf6.regional_statistics(vol, mask, shells_mm=()).rows[-1].region == "zone"
    for bad in ((10.0, 5.0), (0.0,), (float("inf"),), (-1.0,)):
        with pytest.raises(ValueError):
            inf6.regional_statistics(vol, mask, spacing=(1, 1, 1), shells_mm=bad)
    with pytest.raises(ValueError):
        inf6.regional_statistics(vol, mask, zones=0, shells_mm=())
    with pytest.raises(ValueError):
        inf6.regional_statistics(vol, mask, zone_by="area", shells_mm=())
    many = ((np.arange(vol.size) % 60) + 1).astype(np.uint8).reshape(vol.shape)
    with pytest.raises(ValueError, match="region codes"):
        inf6.regional_statistics(vol, many, zones=5, shells_mm=())    # 60 labels x 5 zones > 255
    with pytest.raises(ValueError):
        inf6.regional_statistics(vol, mask[:-1], shells_mm=())
    with pytest.raises(ValueError):
        inf6.regional_statistics(tv, tm[:-1], shells_mm=())
    with pytest.raises(ValueError):
        inf6.regional_statistics(tv, mask, shells_mm=())                # mixed placements
    with pytest.raises(ValueError):
        inf6.surface_distance(mask, (1.0, 0.0, 1.0))
    with pytest.raises(TypeError):
        inf6.surface_distance(mask.astype(np.int16), (1.0, 1.0, 1.0))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            inf6.regional_statistics(tv.to("cuda:1"), tm.to("cuda:1"), shells_mm=())
    # the C entry points refuse bad arguments before any kernel runs
    eng = inf6.engine
    out = torch.empty(mask.shape, dtype=torch.float32, device="cuda:0")
    with pytest.raises(_native.NativeError, match="axis"):
        eng.plane_label_counts_dev(tm.data_ptr(), mask.shape, 3)
    with pytest.raises(_native.NativeError, match="not a CUDA pointer|not device memory"):
        eng.plane_label_counts_dev(mask.ctypes.data, mask.shape, 0)
    with pytest.raises(_native.NativeError, match="spacing"):
        eng.surface_distance_dev(tm.data_ptr(), mask.shape, (1.0, float("nan"), 1.0), out.data_ptr())
    with pytest.raises(_native.NativeError, match="not a CUDA pointer|not device memory"):
        eng.surface_distance_dev(tm.data_ptr(), mask.shape, (1.0, 1.0, 1.0), np.zeros(mask.shape, np.float32).ctypes.data)
    region = torch.empty(mask.shape, dtype=torch.uint8, device="cuda:0")
    lut = np.zeros((mask.shape[0], 256), np.uint8)
    with pytest.raises(_native.NativeError, match="lut_size"):
        eng.region_map_dev(tm.data_ptr(), mask.shape, lut[:-1], region.data_ptr(), axis=0)
    bad = lut.copy()
    bad[3, 0] = 1
    with pytest.raises(_native.NativeError, match="label 0"):
        eng.region_map_dev(tm.data_ptr(), mask.shape, bad, region.data_ptr(), axis=0)
    with pytest.raises(_native.NativeError, match="increasing"):
        eng.region_map_dev(tm.data_ptr(), mask.shape, np.zeros((3, 256), np.uint8), region.data_ptr(), d_dist_ptr=out.data_ptr(),
                           bounds=(5.0, 2.0))
    with pytest.raises(_native.NativeError, match="empty volume"):
        eng.plane_label_counts_dev(tm.data_ptr(), (0, 64, 64), 0)
    # the engine still works after the refusals
    got = inf6.regional_statistics(tv, tm, spacing=(1.0, 1.0, 1.0), percentiles=Q, thresholds=T)
    check_regions(got, vol, mask, (1.0, 1.0, 1.0), 0, True, 3, "volume", (10.0,), Q, T)


@pytest.mark.parametrize("ext", ["json", "csv"])
def test_cli(tmp_path, weights, ext):
    import csv
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    vol = synth.phantom(6, 160, 176, seed=22)
    src = lio.Volume(vol, (0.75, 0.5, 1.5))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = str(tmp_path / ("regions." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", weights[3], "--noprogress", "--batchsize", "4", "--regions", out])
    inf = LMInferer(modelpath=weights[3], tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.regional_statistics(v, inf.apply(v))
    if ext == "json":
        got = json.load(open(out))
        assert got == json.loads(json.dumps(want.to_dict()))
        assert got["zones"] == 3 and got["shells_mm"] == [10.0]
    else:
        rows = list(csv.DictReader(open(out)))
        assert [(r["label"], r["region"], int(r["index"])) for r in rows] == [(str(r.label), r.region, r.index) for r in want.rows]
        for r, w in zip(rows, want.rows):
            assert int(r["voxels"]) == w.stats.voxels
