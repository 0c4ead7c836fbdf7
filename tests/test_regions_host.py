"""Regional statistics without a GPU: the zone rule, the names, the LUTs, the argument checks, the writers and the CLI flag."""
import ctypes as C
import csv
import json
import math

import numpy as np
import pytest


def direct_zones(counts, zones, zone_by, superior_high):
    """The zone rule stated plane by plane in Python integers."""
    n = len(counts)
    order = list(range(n - 1, -1, -1)) if superior_high else list(range(n))
    c = [int(counts[p]) for p in order]
    occ = [i for i in range(n) if c[i]]
    out = [-1] * n
    if not occ:
        return out
    a, b, V = occ[0], occ[-1], sum(c)
    for i in range(a, b + 1):
        if zone_by == "height":
            z = (zones * (i - a)) // (b - a + 1)
        else:
            z = min(zones - 1, (zones * (2 * sum(c[:i]) + c[i])) // (2 * V))
        out[order[i]] = z
    return out


@pytest.mark.parametrize("zone_by", ["volume", "height"])
@pytest.mark.parametrize("superior_high", [True, False])
def test_zone_rule_matches_formula(zone_by, superior_high):
    from lungmask_b200.regions import zone_of_planes
    rng = np.random.default_rng(3)
    cases = [np.zeros(9, np.int64),                                   # absent label
             np.array([0, 0, 0, 17, 0, 0]),                           # a single plane
             np.array([0, 4, 0, 0, 9, 1, 0, 0, 3, 0]),                # empty planes inside the range
             np.array([5]), np.array([1, 1, 1, 1, 1, 1, 1])]
    cases += [rng.integers(0, 3, 40) * rng.integers(0, 5000, 40) for _ in range(20)]
    for c in cases:
        for nz in range(1, 6):
            got = zone_of_planes(c, nz, zone_by, superior_high)
            assert got.tolist() == direct_zones(c, nz, zone_by, superior_high), (c.tolist(), nz)
            inside = got[got >= 0]
            assert inside.size == 0 or (inside.min() >= 0 and inside.max() < nz)


def test_zone_rule_properties():
    from lungmask_b200.regions import zone_of_planes
    c = np.array([0, 10, 10, 10, 10, 10, 10, 0])
    assert zone_of_planes(c, 3, "volume", True).tolist() == [-1, 2, 2, 1, 1, 0, 0, -1]   # zone 0 at the high index
    assert zone_of_planes(c, 3, "volume", False).tolist() == [-1, 0, 0, 1, 1, 2, 2, -1]
    assert zone_of_planes(c, 3, "height", True).tolist() == [-1, 2, 2, 1, 1, 0, 0, -1]
    # volume: a heavy apex plane takes the whole first third
    assert zone_of_planes([0, 1, 1, 30], 3, "volume", True).tolist() == [-1, 2, 2, 1]


def test_orientation_axis_and_names():
    from lungmask_b200 import regions as rg
    assert rg.craniocaudal_axis("LPS") == (0, True)
    assert rg.craniocaudal_axis("RAS") == (0, True)
    assert rg.craniocaudal_axis("PLI") == (0, False)
    assert rg.craniocaudal_axis("LIP") == (1, False)
    assert rg.craniocaudal_axis("SAL") == (2, True)
    assert rg.zone_names(3) == ["upper", "middle", "lower"]
    assert rg.zone_names(2) == ["zone 1 of 2", "zone 2 of 2"]
    assert rg.shell_names((10.0,)) == ["depth 0-10 mm", "depth >= 10 mm"]
    assert rg.shell_names((5.0, 12.5)) == ["depth 0-5 mm", "depth 5-12.5 mm", "depth >= 12.5 mm"]


def test_luts():
    from lungmask_b200 import regions as rg
    zones = {1: np.array([-1, 2, 1, 0]), 3: np.array([1, 1, 0, -1])}
    lut, lung = rg.zone_luts([1, 3], zones, np.array([1, 1, 0, 0]), 3)
    assert lut.shape == (4, 256) and (lut[:, 0] == 0).all() and (lung[:, 0] == 0).all()
    assert lut[:, 1].tolist() == [0, 3, 2, 1] and lut[:, 3].tolist() == [5, 5, 4, 0]
    assert lut[:, 2].sum() == 0 and lung[:, 7].tolist() == [2, 2, 1, 1]
    lut, lung = rg.shell_luts([1, 3], 2)
    assert lut[:, 1].tolist() == [1, 2] and lut[:, 3].tolist() == [3, 4] and lung[:, 255].tolist() == [1, 2]
    with pytest.raises(ValueError, match="region codes"):
        rg.check_code_budget(list(range(1, 65)), 4, "zones")
    rg.check_code_budget(list(range(1, 86)), 3, "zones")                 # 255 codes fit


def test_check_arguments():
    from lungmask_b200.regions import check_arguments
    assert check_arguments(3, "volume", (10.0,), (15.0,), (-950,)) == (3, "volume", (10.0,), (15.0,), (-950,))
    assert check_arguments(2, "height", (), 50, -910)[2] == ()
    assert check_arguments(1, "volume", 7.5, (), ())[2] == (7.5,)
    for bad in (0, 256, -1):
        with pytest.raises(ValueError):
            check_arguments(bad, "volume", (), (), ())
    for bad in (2.0, True, "3"):
        with pytest.raises(TypeError):
            check_arguments(bad, "volume", (), (), ())
    with pytest.raises(ValueError):
        check_arguments(3, "area", (), (), ())
    for bad in ((10.0, 5.0), (5.0, 5.0), (0.0,), (-1.0,), (float("nan"),), (float("inf"),), (1.0, 1.0 + 1e-12)):
        with pytest.raises(ValueError):
            check_arguments(3, "volume", bad, (), ())
    with pytest.raises(ValueError):
        check_arguments(3, "volume", tuple(range(1, 256)), (), ())
    with pytest.raises(ValueError):
        check_arguments(3, "volume", (), (101.0,), ())


def test_null_engine_refused():
    from lungmask_b200 import _native
    L = _native.lib()
    z = np.zeros(257 * 4, np.int64)
    p = C.c_void_p(z.ctypes.data)
    assert L.lm_plane_label_counts_dev(None, p, 1, 1, 1, 0, p, None) == -1
    assert "NULL" in L.lm_last_error().decode()
    assert L.lm_surface_distance_dev(None, p, 1, 1, 1, p, p, None) == -1
    assert L.lm_region_map_dev(None, p, None, 1, 1, 1, 0, None, 0, p, 256, p, None) == -1


def _regional(spacing=(0.5, 0.5, 2.0), shells=(10.0,)):
    from lungmask_b200 import regions as rg
    q, t = (15.0,), (-950,)
    counts = np.zeros((4, 257), np.int64)
    counts[:, 1] = (0, 2, 3, 1)
    counts[:, 256] = counts[:, 1]

    def res(rows):
        r = {"voxels": np.zeros(257, np.int64), "nan_voxels": np.zeros(257, np.int64),
             "moments": np.full((257, 4), np.nan), "percentile": np.full((257, 1), np.nan),
             "below_count": np.zeros((257, 1), np.int64)}
        for code, vox in rows.items():
            r["voxels"][code] = vox
            r["moments"][code] = (-900.0 - code, 10.0, -1000.0, -800.0)
            r["percentile"][code] = -950.5
            r["below_count"][code] = vox // 2
        return r

    lz = {1: rg.zone_of_planes(counts[:, 1], 3, "volume", True)}
    lung = rg.zone_of_planes(counts[:, 256], 3, "volume", True)
    zr, sr = res({1: 1, 2: 3, 3: 2}), res({1: 4, 2: 2})
    return rg.build([1, 2], [1], "R231", spacing, counts, 0, True, 3, "volume", shells, q, t, lz, lung, zr, zr,
                    sr if shells else None, sr if shells else None)


def test_rows_and_dict():
    r = _regional()
    assert [(x.label, x.region, x.index) for x in r.rows] == \
        [(1, "zone", 0), (1, "zone", 1), (1, "zone", 2), (1, "shell", 0), (1, "shell", 1),
         (2, "zone", 0), (2, "zone", 1), (2, "zone", 2), (2, "shell", 0), (2, "shell", 1),
         ("lung", "zone", 0), ("lung", "zone", 1), ("lung", "zone", 2), ("lung", "shell", 0), ("lung", "shell", 1)]
    up = r.row(1, "zone", 0)
    assert up.name == "right lung" and up.region_name == "upper" and up.stats.voxels == 1 and up.planes == (3, 3)
    assert up.stats.volume_ml == 0.5 * 0.5 * 2.0 / 1000.0
    assert r.row(1, "shell", 1).depth_mm == (10.0, math.inf) and r.row(1, "shell", 1).stats.voxels == 2
    assert r.row(2, "zone", 1).stats.voxels == 0 and math.isnan(r.row(2, "zone", 1).stats.mean_hu)
    assert r.profile[1].tolist() == [0, 2, 3, 1]
    d = json.loads(json.dumps(r.to_dict(), allow_nan=False))
    assert d["rows"][4]["depth_mm"] == [10.0, None] and d["profile"]["lung"] == [0, 2, 3, 1]
    assert [x.region for x in _regional(shells=()).rows].count("shell") == 0


def test_save_json_and_csv(tmp_path):
    from lungmask_b200.io import save_regional_statistics
    r = _regional()
    save_regional_statistics(str(tmp_path / "r.json"), r)
    assert json.load(open(tmp_path / "r.json")) == json.loads(json.dumps(r.to_dict()))
    save_regional_statistics(str(tmp_path / "r.csv"), r)
    rows = list(csv.DictReader(open(tmp_path / "r.csv")))
    assert len(rows) == len(r.rows)
    assert rows[0]["region_name"] == "upper" and rows[0]["first_plane"] == "3" and rows[0]["depth_min_mm"] == ""
    assert rows[4]["depth_min_mm"] == "10.0" and rows[4]["depth_max_mm"] == "inf" and rows[4]["first_plane"] == ""
    assert rows[0]["percentile_15"] == "-950.5" and rows[0]["fraction_below_-950"] == "0.0"
    with pytest.raises(SystemExit):
        save_regional_statistics(str(tmp_path / "r.xlsx"), r)


def test_cli_regions_flag(tmp_path):
    from lungmask_b200.__main__ import build_parser, main
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 4, 4), np.int16))
    assert build_parser().parse_args([str(inp), "out.nii", "--regions", "r.json"]).regions == "r.json"
    assert build_parser().parse_args([str(inp), "out.nii"]).regions is None
    with pytest.raises(SystemExit, match="regions"):
        main([str(inp), str(tmp_path / "out.nii"), "--regions", str(tmp_path / "r.xlsx")])
