"""Host side of the LAA cluster size distributions: the pair-count bound, the D fit, the argument checks, the JSON / CSV
writer and the CLI flags."""
import csv
import ctypes as C
import json
import math

import numpy as np
import pytest


def _max_distinct(v):
    """The most distinct positive sizes that sum to at most v: the largest k with k (k + 1) / 2 <= v."""
    k = 0
    while (k + 1) * (k + 2) // 2 <= v:
        k += 1
    return k


def _worst_pairs(n):
    """Brute force: the most (size, count) pairs a volume of n voxels can produce over rows 1..255 (the label rows share
    at most n LAA voxels) plus row 256 (at most n).  DP over the label rows, each row best given its voxel budget."""
    best = [0] * (n + 1)   # best[b]: most pairs from label rows using at most b voxels
    for _ in range(255):
        new = best[:]
        for b in range(n + 1):
            for v in range(1, b + 1):
                c = _max_distinct(v) + best[b - v]
                if c > new[b]:
                    new[b] = c
        if new == best:   # more rows no longer help
            break
        best = new
    return best[n] + _max_distinct(n)


def test_max_pairs_bound():
    from lungmask_b200 import _native
    L = _native.lib()
    for n in list(range(0, 40)) + [63, 64, 65, 100, 120]:
        assert L.lm_laa_max_pairs(n) >= _worst_pairs(n), n
    for k in (1, 2, 3, 1000, 65535, 65536, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1):
        for n in (k * k - 1, k * k, k * k + 1):
            ceil_sqrt = math.isqrt(n) + (math.isqrt(n) ** 2 < n)
            assert L.lm_laa_max_pairs(n) == 32 * ceil_sqrt + 256, n
    assert L.lm_laa_max_pairs(300 * 512 * 512) == 284064   # 4.5 MB of int64 pairs


def test_max_pairs_worst_case_layouts():
    """The bound holds for the densest layout: every row with sizes 1..k, the union with 1..k' on the same voxels."""
    from lungmask_b200 import _native
    L = _native.lib()
    for n in (10, 1000, 100_000, 300 * 512 * 512):
        per_row = n // 255
        pairs = 255 * _max_distinct(per_row) + _max_distinct(n)
        assert pairs <= L.lm_laa_max_pairs(n)


def test_fit_d_matches_polyfit():
    from lungmask_b200.clusters import fit_d
    rng = np.random.default_rng(3)
    for _ in range(20):
        sizes = np.unique(rng.integers(1, 5000, rng.integers(2, 60)))
        counts = rng.integers(1, 1000, sizes.size)
        if sizes.size < 2:
            continue
        y = np.cumsum(counts[::-1])[::-1]
        want = -np.polyfit(np.log10(sizes), np.log10(y), 1)[0]
        assert abs(fit_d(sizes, counts) - want) <= 1e-9 * max(1.0, abs(want))
        m = int(sizes[sizes.size // 2])
        keep = sizes >= m
        if keep.sum() >= 2:
            want_m = -np.polyfit(np.log10(sizes[keep]), np.log10(np.cumsum(counts[keep][::-1])[::-1]), 1)[0]
            assert abs(fit_d(sizes, counts, m) - want_m) <= 1e-9 * max(1.0, abs(want_m))


def test_fit_d_exact_power_law():
    from lungmask_b200.clusters import fit_d
    # Y(s) = 4096 s^-1.5 at s = 1, 4, 16, 64, 256: Y = 4096, 512, 64, 8, 1
    sizes = np.array([1, 4, 16, 64, 256])
    y = np.array([4096, 512, 64, 8, 1])
    counts = y - np.append(y[1:], 0)
    assert abs(fit_d(sizes, counts) - 1.5) < 1e-12
    assert abs(fit_d(sizes[::-1], counts[::-1]) - 1.5) < 1e-12   # order of the pairs does not matter
    assert math.isnan(fit_d([], []))
    assert math.isnan(fit_d([5], [100]))
    assert math.isnan(fit_d(sizes, counts, min_cluster_voxels=257))
    assert math.isnan(fit_d(sizes, counts, min_cluster_voxels=256))   # one point left


def test_check_arguments():
    from lungmask_b200.clusters import check_arguments
    assert check_arguments(-950, 6, 1) == (-950, 6, 1)
    assert check_arguments(-950.0, np.int64(26), 3) == (-950, 26, 3)
    assert check_arguments(-1024, 4, 1) == (-1024, 4, 1) and check_arguments(3072, 4, 1)[0] == 3072
    for t in (-1025, 3073):
        with pytest.raises(ValueError):
            check_arguments(t, 6, 1)
    for c in (0, 5, 8, 18, 27):
        with pytest.raises(ValueError):
            check_arguments(-950, c, 1)
    with pytest.raises(ValueError):
        check_arguments(-950, 6, 0)
    for bad in (-950.5, "x", None, True):
        with pytest.raises(TypeError):
            check_arguments(bad, 6, 1)


def test_null_engine_refused_dev():
    from lungmask_b200 import _native
    L = _native.lib()
    z = np.zeros(257, np.int64)
    p = C.c_void_p(z.ctypes.data)
    assert L.lm_laa_clusters_dev(None, p, 0, p, 1, 1, 1, -950, 6, p, p, p, p, p, 1000, None) == -1
    assert "NULL" in L.lm_last_error().decode()


def _clusters(spacing=(0.5, 0.5, 2.0)):
    from lungmask_b200 import clusters as cl
    res = {k: np.zeros(257, np.int64) for k in ("laa_voxels", "n_clusters", "n_pairs")}
    # row 1: sizes 1 x 5, 2 x 2, 10 x 1; row 256 the same plus one of 4
    res["laa_voxels"][[1, 256]] = (19, 23)
    res["n_clusters"][[1, 256]] = (8, 9)
    res["n_pairs"][[1, 256]] = (3, 4)
    res["sizes"] = np.array([1, 2, 10, 1, 2, 4, 10], np.int64)
    res["counts"] = np.array([5, 2, 1, 5, 2, 1, 1], np.int64)
    res["offsets"] = np.concatenate([[0], np.cumsum(res["n_pairs"])])
    return cl.from_native(res, {1, 2}, "R231", spacing, -950, 6, 1)


def test_rows():
    from lungmask_b200.clusters import fit_d
    s = _clusters()
    assert [r.label for r in s.rows] == [1, 2, "lung"] and s[1].name == "right lung" and s["lung"].name == "lung"
    assert s[1].laa_voxels == 19 and s[1].clusters == 8 and s[1].largest_voxels == 10
    assert s[1].laa_volume_ml == 19 * 0.5 / 1000.0 and s[1].largest_ml == 10 * 0.5 / 1000.0
    assert s[1].sizes.tolist() == [1, 2, 10] and s[1].counts.tolist() == [5, 2, 1]
    assert s[1].d == fit_d([1, 2, 10], [5, 2, 1])
    assert s["lung"].sizes.tolist() == [1, 2, 4, 10]
    assert s[2].laa_voxels == 0 and s[2].largest_voxels == 0 and math.isnan(s[2].d) and s[2].sizes.size == 0
    with pytest.raises(KeyError):
        s[3]
    assert _clusters(None)[1].laa_volume_ml is None and _clusters(None)[1].largest_ml is None


def test_save_json_and_csv(tmp_path):
    from lungmask_b200 import io as lio
    s = _clusters()
    pj, pc = str(tmp_path / "c.json"), str(tmp_path / "c.csv")
    lio.save_clusters(pj, s)
    d = json.load(open(pj))
    assert d["spacing"] == [0.5, 0.5, 2.0] and d["threshold"] == -950 and d["connectivity"] == 6
    assert d["min_cluster_voxels"] == 1
    assert [r["label"] for r in d["rows"]] == [1, 2, "lung"]
    assert d["rows"][0]["sizes"] == [1, 2, 10] and d["rows"][0]["counts"] == [5, 2, 1]
    assert d["rows"][1]["d"] is None and d["rows"][1]["sizes"] == []   # NaN -> null
    lio.save_clusters(pc, s)
    rows = list(csv.DictReader(open(pc)))
    assert list(rows[0].keys()) == ["label", "name", "laa_voxels", "laa_volume_ml", "clusters", "largest_voxels", "largest_ml", "d"]
    assert rows[0]["name"] == "right lung" and int(rows[0]["clusters"]) == 8 and float(rows[0]["d"]) == s[1].d
    assert rows[1]["d"] == "nan" and rows[2]["label"] == "lung"
    lio.save_clusters(str(tmp_path / "n.csv"), _clusters(None))
    assert list(csv.DictReader(open(str(tmp_path / "n.csv"))))[0]["laa_volume_ml"] == ""
    with pytest.raises(SystemExit):
        lio.save_clusters(str(tmp_path / "c.txt"), s)


def test_cli_clusters_flags(tmp_path):
    from lungmask_b200.__main__ import build_parser, main
    inp = tmp_path / "v.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    args = build_parser().parse_args([str(inp), "out.nii", "--clusters", "c.json", "--clusters-threshold", "-910",
                                      "--clusters-connectivity", "26"])
    assert (args.clusters, args.clusters_threshold, args.clusters_connectivity) == ("c.json", -910, 26)
    args = build_parser().parse_args([str(inp), "out.nii"])
    assert (args.clusters, args.clusters_threshold, args.clusters_connectivity) == (None, -950, 6)
    with pytest.raises(SystemExit):
        build_parser().parse_args([str(inp), "out.nii", "--clusters-connectivity", "8"])
    # refused before any model is loaded
    with pytest.raises(SystemExit, match="clusters"):
        main([str(inp), str(tmp_path / "out.nii"), "--clusters", str(tmp_path / "c.xlsx")])
    with pytest.raises(SystemExit, match="threshold"):
        main([str(inp), str(tmp_path / "out.nii"), "--clusters", str(tmp_path / "c.json"), "--clusters-threshold", "-2000"])
