"""Host side of the texture features (lungmask_b200.texture): the fixed-bin-width discretisation against np.digitize,
the GLCM and GLSZM feature functions against known answers and against a naive loop restatement written here, direction
invariance, argument checks and the JSON / CSV writers.  No GPU."""
import csv
import json
import math

import numpy as np
import pytest

from lungmask_b200 import texture as tx

EPS = np.spacing(1)


# ---- discretisation ----------------------------------------------------------------------------------------------------
def digitize_reference(x, bw):
    """The PyRadiomics binning: np.digitize on the edges min - min % bw, ..., max + bw."""
    x = np.asarray(x)
    mn, mx = x.min(), x.max()
    edges = np.arange(mn - mn % bw, mx + 2 * bw, bw)
    return np.digitize(x, edges)


@pytest.mark.parametrize("dtype", [np.int16, np.float32, np.float64])
@pytest.mark.parametrize("bw", [1, 3, 10, 25])
def test_discretisation_equals_digitize(dtype, bw):
    rng = np.random.default_rng(7 + bw)
    for lo, hi in ((-1024, 300), (-37, 90), (5, 400)):
        x = rng.uniform(lo, hi, 4000)
        if np.dtype(dtype).kind == "i":
            x = np.round(x)
        x = x.astype(dtype)
        # values on bin edges and one ulp below them
        edges = np.arange(bw * (int(np.floor(float(x.min()))) // bw), float(x.max()), bw)[:50].astype(dtype)
        extra = [edges]
        if np.dtype(dtype).kind == "f":
            extra.append(np.nextafter(edges, dtype(-np.inf)).astype(dtype))
        x = np.concatenate([x] + extra)
        x = x[(x >= x.min()) & (x <= x.max())]
        want = digitize_reference(x, bw)
        got = tx.levels(x, bw)
        np.testing.assert_array_equal(got, want)
        if want.max() > 255:
            with pytest.raises(ValueError, match="more than 255"):
                tx.discretisation(float(x.min()), float(x.max()), bw)
            continue
        low, ng = tx.discretisation(float(x.min()), float(x.max()), bw)
        assert ng == int(want.max()) and int(got.min()) == 1
        assert low == bw * (math.floor(float(x.min())) // bw)   # floor(min / bw), without min / bw underflowing


def test_discretisation_negative_minimum_exact():
    assert tx.discretisation(-1024.0, 3071.0, 25) == (-1025, 164)
    assert tx.discretisation(-1000.5, -1000.5, 25) == (-1025, 1)
    assert tx.discretisation(-25.0, -0.25, 25) == (-25, 1)
    assert tx.discretisation(-25.0, 0.0, 25) == (-25, 2)
    np.testing.assert_array_equal(tx.levels(np.array([-25.0, -0.25, 0.0, 24.999]), 25), [1, 1, 2, 2])


def test_argument_errors():
    for bad in (0, -3):
        with pytest.raises(ValueError):
            tx.check_arguments(bad)
    for bad in (2.5, "25", True, None):
        with pytest.raises(TypeError):
            tx.check_arguments(bad)
    assert tx.check_arguments(25.0) == 25 and tx.check_arguments(np.int64(10)) == 10
    with pytest.raises(ValueError, match="more than 255.*larger bin width"):
        tx.discretisation(-1024.0, 3071.0, 5, "row 1")
    tx.discretisation(-1024.0, -1024.0 + 254 * 5, 5)   # exactly 255 levels
    with pytest.raises(ValueError, match="non-finite"):
        tx.discretisation(-np.inf, 0.0, 25)
    with pytest.raises(ValueError, match="non-finite"):
        tx.discretisation(0.0, np.inf, 25)


def test_suggested_bin_width_suffices():
    with pytest.raises(ValueError) as ex:
        tx.discretisation(-1024.0, 3071.0, 5)
    wider = int(str(ex.value).split("(")[-1].split()[0])
    assert tx.discretisation(-1024.0, 3071.0, wider)[1] <= 255
    with pytest.raises(ValueError):
        tx.discretisation(-1024.0, 3071.0, wider - 1)


# ---- naive restatement -------------------------------------------------------------------------------------------------
def naive_glcm_direction(P, ng):
    tot = sum(P[a][b] for a in range(ng) for b in range(ng))
    p = [[P[a][b] / tot for b in range(ng)] for a in range(ng)]
    px = [sum(p[a][b] for b in range(ng)) for a in range(ng)]
    mu = sum((a + 1) * px[a] for a in range(ng))
    sx2 = sum((a + 1 - mu) ** 2 * px[a] for a in range(ng))
    psum = {k: 0.0 for k in range(2, 2 * ng + 1)}
    pdiff = {k: 0.0 for k in range(ng)}
    for a in range(ng):
        for b in range(ng):
            psum[a + b + 2] += p[a][b]
            pdiff[abs(a - b)] += p[a][b]
    lg = math.log2
    hx = -sum(px[a] * lg(px[a] + EPS) for a in range(ng))
    hxy = -sum(p[a][b] * lg(p[a][b] + EPS) for a in range(ng) for b in range(ng))
    hxy1 = -sum(p[a][b] * lg(px[a] * px[b] + EPS) for a in range(ng) for b in range(ng))
    hxy2 = -sum(px[a] * px[b] * lg(px[a] * px[b] + EPS) for a in range(ng) for b in range(ng))
    da = sum(k * v for k, v in pdiff.items())
    cells = [(a + 1, b + 1, p[a][b]) for a in range(ng) for b in range(ng)]
    return {
        "Autocorrelation": sum(i * j * q for i, j, q in cells),
        "JointAverage": mu,
        "ClusterProminence": sum((i + j - 2 * mu) ** 4 * q for i, j, q in cells),
        "ClusterShade": sum((i + j - 2 * mu) ** 3 * q for i, j, q in cells),
        "ClusterTendency": sum((i + j - 2 * mu) ** 2 * q for i, j, q in cells),
        "Contrast": sum((i - j) ** 2 * q for i, j, q in cells),
        "Correlation": 1.0 if sx2 == 0 else sum((i - mu) * (j - mu) * q for i, j, q in cells) / sx2,
        "DifferenceAverage": da,
        "DifferenceEntropy": -sum(v * lg(v + EPS) for v in pdiff.values()),
        "DifferenceVariance": sum((k - da) ** 2 * v for k, v in pdiff.items()),
        "JointEnergy": sum(q * q for _, _, q in cells),
        "JointEntropy": hxy,
        "Imc1": 0.0 if hx == 0 else (hxy - hxy1) / hx,
        "Imc2": 0.0 if hxy2 <= hxy else math.sqrt(1 - math.exp(-2 * (hxy2 - hxy))),
        "Idm": sum(v / (1 + k * k) for k, v in pdiff.items()),
        "Idmn": sum(v / (1 + k * k / ng ** 2) for k, v in pdiff.items()),
        "Id": sum(v / (1 + k) for k, v in pdiff.items()),
        "Idn": sum(v / (1 + k / ng) for k, v in pdiff.items()),
        "InverseVariance": sum(v / k ** 2 for k, v in pdiff.items() if k >= 1),
        "MaximumProbability": max(q for _, _, q in cells),
        "SumEntropy": -sum(v * lg(v + EPS) for v in psum.values()),
        "SumSquares": sx2,
    }


def naive_glcm(U, ng):
    per = []
    for u in U:
        P = [[0.0] * ng for _ in range(ng)]
        t = 0
        for a in range(ng):
            for b in range(a, ng):
                P[a][b] += u[t]
                P[b][a] += u[t]
                t += 1
        if sum(map(sum, P)):
            per.append(naive_glcm_direction(P, ng))
    return {k: sum(f[k] for f in per) / len(per) for k in tx.GLCM_FEATURES}


def naive_glszm(zones, n_voxels):
    nz = sum(c for _, _, c in zones)
    by_l, by_s = {}, {}
    for l, s, c in zones:
        by_l[l] = by_l.get(l, 0) + c
        by_s[s] = by_s.get(s, 0) + c
    mi = sum(l * c for l, _, c in zones) / nz
    ms = sum(s * c for _, s, c in zones) / nz
    return {
        "SmallAreaEmphasis": sum(c / s ** 2 for _, s, c in zones) / nz,
        "LargeAreaEmphasis": sum(c * s ** 2 for _, s, c in zones) / nz,
        "GrayLevelNonUniformity": sum(v ** 2 for v in by_l.values()) / nz,
        "GrayLevelNonUniformityNormalized": sum(v ** 2 for v in by_l.values()) / nz ** 2,
        "SizeZoneNonUniformity": sum(v ** 2 for v in by_s.values()) / nz,
        "SizeZoneNonUniformityNormalized": sum(v ** 2 for v in by_s.values()) / nz ** 2,
        "ZonePercentage": nz / n_voxels,
        "GrayLevelVariance": sum(c / nz * (l - mi) ** 2 for l, _, c in zones),
        "ZoneVariance": sum(c / nz * (s - ms) ** 2 for _, s, c in zones),
        "ZoneEntropy": -sum(c / nz * math.log2(c / nz + EPS) for _, _, c in zones),
        "LowGrayLevelZoneEmphasis": sum(c / l ** 2 for l, _, c in zones) / nz,
        "HighGrayLevelZoneEmphasis": sum(c * l ** 2 for l, _, c in zones) / nz,
        "SmallAreaLowGrayLevelEmphasis": sum(c / (l ** 2 * s ** 2) for l, s, c in zones) / nz,
        "SmallAreaHighGrayLevelEmphasis": sum(c * l ** 2 / s ** 2 for l, s, c in zones) / nz,
        "LargeAreaLowGrayLevelEmphasis": sum(c * s ** 2 / l ** 2 for l, s, c in zones) / nz,
        "LargeAreaHighGrayLevelEmphasis": sum(c * l ** 2 * s ** 2 for l, s, c in zones) / nz,
    }


def numpy_matrices(L):
    """U (13, T) and the GLSZM triples of a small level map (0 = outside), by slicing and scipy.ndimage.label."""
    import scipy.ndimage as ndi
    ng = int(L.max())
    T = ng * (ng + 1) // 2
    U = np.zeros((13, T), np.int64)
    n = L.shape
    for d, off in enumerate(tx.OFFSETS):
        src = tuple(slice(max(0, -o), n[k] - max(0, o)) for k, o in enumerate(off))
        dst = tuple(slice(max(0, o), n[k] - max(0, -o)) for k, o in enumerate(off))
        a, b = L[src].astype(np.int64), L[dst].astype(np.int64)
        both = (a > 0) & (b > 0)
        i, j = np.minimum(a, b)[both], np.maximum(a, b)[both]
        idx = (i - 1) * ng - (i - 1) * (i - 2) // 2 + (j - i)
        U[d] = np.bincount(idx, minlength=T)
    zones = []
    for lv in range(1, ng + 1):
        lab, k = ndi.label(L == lv, np.ones((3, 3, 3), bool))
        if k:
            s, c = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
            zones += [(lv, int(a), int(b)) for a, b in zip(s, c)]
    return U, np.array(zones, np.int64).reshape(-1, 3)


def assert_close(got, want, tol=1e-12):
    for k, w in want.items():
        g = got[k]
        assert (math.isnan(g) and math.isnan(w)) or abs(g - w) <= tol * max(1.0, abs(w)), (k, g, w)


# ---- known answers -----------------------------------------------------------------------------------------------------
def test_checkerboard_known_answers():
    """A two-level checkerboard along x in one row: every x-pair is (1, 2)."""
    L = np.array([[[1, 2, 1, 2, 1, 2]]], np.uint8)
    U, zones = numpy_matrices(L)
    assert U[0].tolist() == [0, 5, 0] and not U[1:].any()
    f = tx.glcm_features(U, 2)
    # P = [[0, 5], [5, 0]] / 10
    assert f["Contrast"] == 1.0 and f["JointAverage"] == 1.5 and f["Autocorrelation"] == 2.0
    assert f["Correlation"] == -1.0 and f["JointEnergy"] == 0.5 and f["MaximumProbability"] == 0.5
    assert f["DifferenceAverage"] == 1.0 and f["DifferenceVariance"] == 0.0 and f["InverseVariance"] == 1.0
    assert abs(f["JointEntropy"] - 1.0) < 1e-12 and f["ClusterTendency"] == 0.0 and f["SumSquares"] == 0.25
    assert f["Id"] == 0.5 and f["Idm"] == 0.5 and f["Idn"] == 2.0 / 3.0
    g = tx.glszm_features(zones[:, 0], zones[:, 1], zones[:, 2], 6)
    assert zones.tolist() == [[1, 1, 3], [2, 1, 3]]
    assert g["SmallAreaEmphasis"] == 1.0 and g["ZonePercentage"] == 1.0 and g["GrayLevelNonUniformity"] == 3.0
    assert g["GrayLevelVariance"] == 0.25 and g["ZoneVariance"] == 0.0


def test_constant_roi():
    L = np.zeros((4, 5, 6), np.uint8)
    L[1:3, 1:4, 1:5] = 3
    U, zones = numpy_matrices(L)
    f = tx.glcm_features(U, 3)
    assert f["Correlation"] == 1.0 and f["Imc1"] == 0.0 and f["Imc2"] == 0.0 and f["Contrast"] == 0.0
    assert f["JointEnergy"] == 1.0 and f["JointAverage"] == 3.0 and f["MaximumProbability"] == 1.0
    assert zones.tolist() == [[3, 24, 1]]
    g = tx.glszm_features(zones[:, 0], zones[:, 1], zones[:, 2], 24)
    assert g["ZonePercentage"] == 1 / 24 and g["LargeAreaEmphasis"] == 576.0 and g["GrayLevelVariance"] == 0.0


def test_no_pairs_and_no_zones():
    U = np.zeros((13, 6), np.int64)
    assert all(math.isnan(v) for v in tx.glcm_features(U, 3).values())
    assert all(math.isnan(v) for v in tx.glszm_features([], [], [], 0).values())
    row = tx.build_row(4, "label 4", 0, 25)
    assert row.voxels == 0 and row.low is None and row.n_levels == 0 and math.isnan(row.glcm["Contrast"])
    one = np.zeros((3, 3, 3), np.uint8)
    one[1, 1, 1] = 1
    U1, z1 = numpy_matrices(one)
    r = tx.build_row(1, "x", 1, 25, -1000, 1, U1, z1)
    assert all(math.isnan(v) for v in r.glcm.values()) and r.glszm["ZonePercentage"] == 1.0


# ---- against the naive restatement -------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_features_match_naive_loops(seed):
    rng = np.random.default_rng(seed)
    ng = int(rng.integers(3, 9))
    L = rng.integers(0, ng + 1, (5, 6, 7)).astype(np.uint8)
    L[L == 0] = rng.integers(0, 2, int((L == 0).sum())).astype(np.uint8)   # some holes
    L[0, 0, 0] = ng
    U, zones = numpy_matrices(L)
    assert_close(tx.glcm_features(U, ng), naive_glcm(U, ng))
    n = int((L > 0).sum())
    assert_close(tx.glszm_features(zones[:, 0], zones[:, 1], zones[:, 2], n), naive_glszm(zones.tolist(), n))


def test_direction_permutation_invariance():
    """A flip or a transpose of the volume permutes the 13 direction matrices: the features stay within 1e-12."""
    rng = np.random.default_rng(11)
    L = np.clip(np.round(rng.normal(4, 1.5, (6, 7, 8))), 0, 8).astype(np.uint8)
    L[0, 0, 0] = 8
    U, _ = numpy_matrices(L)
    want = tx.glcm_features(U, 8)
    for V in (L[::-1], L[:, ::-1], L[:, :, ::-1], L.transpose(0, 2, 1).copy(), L.transpose(2, 1, 0).copy()):
        U2, _ = numpy_matrices(np.ascontiguousarray(V))
        assert sorted(map(tuple, U2)) == sorted(map(tuple, U))
        assert_close(tx.glcm_features(U2, 8), want)
    perm = rng.permutation(13)
    assert_close(tx.glcm_features(U[perm], 8), want)


# ---- writers -----------------------------------------------------------------------------------------------------------
def _features():
    rng = np.random.default_rng(5)
    L = rng.integers(0, 5, (4, 5, 6)).astype(np.uint8)
    L[0, 0, 0] = 4
    U, zones = numpy_matrices(L)
    rows = [tx.build_row(1, "right lung", int((L > 0).sum()), 25, -1000, 4, U, zones), tx.build_row(2, "left lung", 0, 25),
            tx.build_row(256, "lung", int((L > 0).sum()), 25, -1000, 4, U, zones)]
    return tx.TextureFeatures((0.7, 0.7, 1.25), 25, rows)


def test_save_json_and_csv(tmp_path):
    from lungmask_b200.io import save_texture
    res = _features()
    assert res["lung"].label == "lung" and res[2].voxels == 0
    with pytest.raises(KeyError):
        res[3]
    p = str(tmp_path / "t.json")
    save_texture(p, res)
    got = json.load(open(p))
    assert got == json.loads(json.dumps(res.to_dict()))
    assert got["bin_width"] == 25 and got["rows"][1]["glcm"]["Contrast"] is None
    assert got["rows"][0]["glszm_zones"] == res[1].zones.tolist()
    p = str(tmp_path / "t.csv")
    save_texture(p, res)
    rows = list(csv.DictReader(open(p)))
    assert [r["label"] for r in rows] == ["1", "2", "lung"]
    assert set("glcm_" + k for k in tx.GLCM_FEATURES) <= set(rows[0]) and set("glszm_" + k for k in tx.GLSZM_FEATURES) <= set(rows[0])
    assert float(rows[0]["glcm_Contrast"]) == res[1].glcm["Contrast"] and rows[1]["glcm_Contrast"] == "nan"
    assert rows[1]["low"] == "" and int(rows[0]["n_levels"]) == 4
    with pytest.raises(SystemExit):
        save_texture(str(tmp_path / "t.txt"), res)


def test_cli_checks_bin_width_before_loading(tmp_path):
    from lungmask_b200.__main__ import main
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    with pytest.raises(SystemExit, match="texture-bin-width"):
        main([str(inp), str(tmp_path / "m.npy"), "--texture", str(tmp_path / "t.json"), "--texture-bin-width", "0"])
    with pytest.raises(SystemExit, match="unsupported texture output"):
        main([str(inp), str(tmp_path / "m.npy"), "--texture", str(tmp_path / "t.xlsx")])
