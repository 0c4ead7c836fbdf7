"""Mesh shape features on the host (lungmask_b200.shape): the generated triangle table, closed meshes, the count / corner-sum
formula against a triangle-by-triangle sum, analytic cases, the diameter pruning against brute force, the principal axes
against PyRadiomics' formula restated with numpy, and the argument checks of LMInferer.shape and --shape."""
import collections
import json
import math
import types

import numpy as np
import pytest

from lungmask_b200 import shape as sh

SPACINGS = ((1.0, 1.0, 1.0), (0.703125, 0.703125, 1.25), (0.7, 1.3, 2.5))


def random_mask(seed, shape, labels):
    """Blobs of `labels` labels: smoothed noise thresholded, so that rows have holes, handles and thin parts."""
    import scipy.ndimage as ndi
    rng = np.random.default_rng(seed)
    field = ndi.gaussian_filter(rng.standard_normal(shape), 1.2)
    m = (field > np.quantile(field, 0.45)).astype(np.uint8)
    if labels > 1:
        region = ndi.gaussian_filter(rng.standard_normal(shape), 2.0)
        cuts = np.quantile(region, np.linspace(0, 1, labels + 1)[1:-1])
        m *= (np.searchsorted(cuts, region) + 1).astype(np.uint8)
    return m


def explicit_mesh(member):
    """(triangles as (t, 3, 3) doubled integer vertex coordinates) of a boolean row, cube by cube from the table."""
    M = np.pad(np.asarray(member, bool), 1)
    n0, n1, n2 = member.shape
    conf = np.zeros((n0 + 1, n1 + 1, n2 + 1), np.int64)
    for k, (d0, d1, d2) in enumerate(sh.CORNERS):
        conf |= M[d0:d0 + n0 + 1, d1:d1 + n1 + 1, d2:d2 + n2 + 1].astype(np.int64) << k
    tris = []
    for p in np.argwhere((conf != 0) & (conf != 255)):
        for t in sh.TRIANGLES[conf[tuple(p)]]:
            tris.append([2 * (p - 1) + sh.EDGE_MID2[e] for e in t])
    return np.array(tris, np.int64).reshape(-1, 3, 3)


def triangle_sums(tris, spacing):
    """(area, volume) triangle by triangle, vertices in (x, y, z) mm."""
    sx, sy, sz = spacing
    P = tris[..., ::-1].astype(np.float64) * (0.5 * np.array([sx, sy, sz]))
    a, b, c = P[:, 0], P[:, 1], P[:, 2]
    area = 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum()
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0
    return float(area), float(vol)


def area_volume(member, spacing):
    counts, possum, _ = sh.cube_sums_host(np.asarray(member, np.uint8))
    return sh.mesh_area_volume(counts[1], possum[1], spacing)


# ---- table ------------------------------------------------------------------------------------------------------------
def test_table_loops_closed_and_oriented():
    assert sh.TRIANGLES[0] == [] and sh.TRIANGLES[255] == []
    for c in range(256):
        lps = sh.loops(c)   # raises when a segment chain does not close or an edge starts two segments
        inside = [(c >> k) & 1 for k in range(8)]
        crossing = {e for e, (a, b, _) in enumerate(sh.EDGES) if inside[a] != inside[b]}
        seen = [e for lp in lps for e in lp]
        assert sorted(seen) == sorted(crossing), c
        assert all(lp[0] == min(lp) for lp in lps)
        assert len(sh.TRIANGLES[c]) <= 5
        if bin(c).count("1") in (1, 7):   # one corner cut off: one triangle
            assert len(sh.TRIANGLES[c]) == 1


def test_table_is_generated_deterministically():
    assert sh.triangle_table() == sh.TRIANGLES
    assert max(len(t) for t in sh.TRIANGLES) == 5


# ---- closed meshes and the sums formula -------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,shape,labels", [(0, (9, 11, 13), 1), (1, (14, 12, 10), 3), (2, (20, 20, 20), 6),
                                               (3, (7, 19, 16), 2), (4, (16, 16, 16), 4)])
def test_random_meshes_closed_and_sums_formula(seed, shape, labels):
    m = random_mask(seed, shape, labels)
    counts, possum, moments = sh.cube_sums_host(m)
    for r in [int(x) for x in np.unique(m) if x] + [256]:
        member = (m != 0) if r == 256 else (m == r)
        tris = explicit_mesh(member)
        directed = collections.Counter()
        for t in tris:
            for a, b in ((0, 1), (1, 2), (2, 0)):
                directed[(tuple(t[a]), tuple(t[b]))] += 1
        assert max(directed.values()) == 1, (seed, r)
        assert all((b, a) in directed for a, b in directed), (seed, r)
        for sp in SPACINGS:
            A_t, V_t = triangle_sums(tris, sp)
            A, V = sh.mesh_area_volume(counts[r], possum[r], sp)
            assert V > 0 and V_t > 0, (seed, r, sp)
            assert A == pytest.approx(A_t, rel=1e-12) and V == pytest.approx(V_t, rel=1e-12), (seed, r, sp)
        assert moments[r][0] == member.sum()


# ---- analytic cases ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spacing", SPACINGS + ((0.5, 3.0, 1.75),))
def test_single_voxel_octahedron(spacing):
    m = np.zeros((3, 4, 5), np.uint8)
    m[1, 2, 3] = 1
    A, V = area_volume(m, spacing)
    a = [s / 2 for s in spacing]
    assert V == pytest.approx(spacing[0] * spacing[1] * spacing[2] / 6, rel=1e-12)
    assert A == pytest.approx(4 * math.sqrt(a[0] ** 2 * a[1] ** 2 + a[1] ** 2 * a[2] ** 2 + a[2] ** 2 * a[0] ** 2), rel=1e-12)
    d2 = sh.max_diameters_host(m > 0, spacing)
    sx, sy, sz = spacing
    assert math.sqrt(d2[0]) == pytest.approx(max(spacing), rel=1e-15)
    assert math.sqrt(d2[1]) == pytest.approx(max(sx, sy), rel=1e-15)   # equal axis-0 (z) index: the x-y plane
    np.testing.assert_array_equal(d2, sh.max_diameters_brute(m > 0, spacing))
    counts, possum, moments = sh.cube_sums_host(m)
    f = sh.features(1, counts[1], possum[1], moments[1], d2, spacing)
    assert math.isnan(f["MajorAxisLength"]) is False and f["MajorAxisLength"] == 0.0
    assert math.isnan(f["Elongation"]) and math.isnan(f["Flatness"])


@pytest.mark.parametrize("a,b,c", [(4, 5, 6), (1, 1, 1), (2, 7, 3), (1, 6, 1)])
def test_box(a, b, c):
    m = np.zeros((a + 2, b + 3, c + 1), np.uint8)
    m[1:1 + a, 2:2 + b, 0:c] = 1   # touches the last face of axis 2: closed there by the padding
    A, V = area_volume(m, (1.0, 1.0, 1.0))
    assert V == pytest.approx(a * b * c - (a + b + c - 3) / 2 - 5 / 6, rel=1e-12, abs=1e-12)
    want = 2 * ((a - 1) * (b - 1) + (b - 1) * (c - 1) + (c - 1) * (a - 1)) + 2 * math.sqrt(2) * (a + b + c - 3) + math.sqrt(3)
    assert A == pytest.approx(want, rel=1e-12)
    if (a, b, c) == (4, 5, 6):
        assert round(V, 4) == 113.1667 and round(A, 4) == 129.6732


def test_ball():
    r = 12
    z, y, x = np.ogrid[-r - 2:r + 3, -r - 2:r + 3, -r - 2:r + 3]
    m = (x * x + y * y + z * z <= r * r).astype(np.uint8)
    A, V = area_volume(m, (1.0, 1.0, 1.0))
    assert V == pytest.approx(4 / 3 * math.pi * r ** 3, rel=0.02)
    assert A == pytest.approx(4 * math.pi * r ** 2, rel=0.08)
    counts, possum, moments = sh.cube_sums_host(m)
    f = sh.features(int(m.sum()), counts[1], possum[1], moments[1], sh.max_diameters_host(m > 0, (1, 1, 1), hull=True),
                    (1.0, 1.0, 1.0))
    assert 0.9 < f["Sphericity"] < 1.0
    assert f["Maximum3DDiameter"] == pytest.approx(2 * r + 1, abs=1.0)
    assert f["Elongation"] == pytest.approx(1.0, abs=1e-9) and f["Flatness"] == pytest.approx(1.0, abs=1e-9)


# ---- diameters --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_pruned_diameters_equal_brute_force(seed):
    m = random_mask(100 + seed, (8 + seed, 10, 9 + 2 * seed), 1 + seed % 3)
    for r in [int(x) for x in np.unique(m) if x] + [256]:
        member = (m != 0) if r == 256 else (m == r)
        for sp in SPACINGS:
            np.testing.assert_array_equal(sh.max_diameters_host(member, sp), sh.max_diameters_brute(member, sp),
                                          err_msg="%s %s %s" % (seed, r, sp))


def _hull_brute(member, spacing):
    """Brute force over the mesh vertices reduced to their convex hull's vertices (per plane for the 2-D families)."""
    V = sh.mesh_vertices(member)
    out = [sh.pair_max_d2(sh._hull_vertices(V, None), spacing)]
    for a in range(3):
        out.append(max(sh.pair_max_d2(sh._hull_vertices(V[V[:, a] == c], a), spacing) for c in np.unique(V[:, a])))
    return np.array(out)


@pytest.mark.parametrize("seed", range(3))
def test_pruned_diameters_equal_hull_brute_force(seed):
    m = random_mask(200 + seed, (30, 34, 38), 2)
    sp = SPACINGS[seed % 2]   # dyadic: every d^2 exact
    for r in (1, 2, 256):
        member = (m != 0) if r == 256 else (m == r)
        want = _hull_brute(member, sp)
        np.testing.assert_array_equal(sh.max_diameters_host(member, sp), want)
        np.testing.assert_array_equal(sh.max_diameters_host(member, sp, hull=True), want)


# ---- principal axes ---------------------------------------------------------------------------------------------------
def pyradiomics_eigenvalues(member, spacing):
    """PyRadiomics' shape.py: physical coordinates, centred, divided by sqrt(Np), X^T X, eigenvalues sorted."""
    s = np.array(spacing[::-1], np.float64)
    coords = np.argwhere(member).astype(np.float64) * s
    Np = len(coords)
    X = (coords - coords.mean(axis=0)) / math.sqrt(Np)
    ev = np.sort(np.linalg.eigvals(X.T @ X).real)
    ev[(ev < 0) & (ev > -1e-10)] = 0
    return ev


@pytest.mark.parametrize("seed", range(4))
def test_principal_axes_match_pyradiomics_formula(seed):
    m = random_mask(300 + seed, (12, 15, 17), 3)
    _, _, moments = sh.cube_sums_host(m)
    for r in [int(x) for x in np.unique(m) if x] + [256]:
        member = (m != 0) if r == 256 else (m == r)
        for sp in SPACINGS:
            got = np.array(sh.principal_moments(moments[r], sp))
            want = pyradiomics_eigenvalues(member, sp)
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * want[-1])


def test_moments_exact():
    m = random_mask(7, (9, 10, 11), 3)
    _, _, moments = sh.cube_sums_host(m)
    for r in [1, 2, 3, 256]:
        idx = np.argwhere((m != 0) if r == 256 else (m == r)).astype(np.int64)
        i, j, k = idx.T
        want = [len(idx), i.sum(), j.sum(), k.sum(), (i * i).sum(), (j * j).sum(), (k * k).sum(), (i * j).sum(),
                (i * k).sum(), (j * k).sum()]
        assert list(moments[r]) == want
    assert not moments[0].any() and not moments[4:256].any()


# ---- results and argument checks --------------------------------------------------------------------------------------
def _features_of(m, spacing):
    counts, possum, moments = sh.cube_sums_host(m)
    rows = []
    for r in [int(x) for x in np.unique(m) if x] + [256]:
        member = (m != 0) if r == 256 else (m == r)
        rows.append(sh.build_row(r, "row", spacing, counts[r], possum[r], moments[r], sh.max_diameters_host(member, spacing)))
    rows.append(sh.build_row(9, "absent", spacing, counts[9], possum[9], moments[9], np.zeros(4)))
    return sh.ShapeFeatures(spacing, rows)


def test_result_objects_and_writer(tmp_path):
    from lungmask_b200.io import save_shape
    m = random_mask(11, (10, 12, 14), 2)
    res = _features_of(m, (0.7, 0.8, 2.0))
    assert res["lung"].voxels == int((m != 0).sum()) and res["lung"]["SurfaceArea"] > 0
    assert all(math.isnan(v) for v in res[9].features.values())
    with pytest.raises(KeyError):
        res[3]
    d = res.to_dict()
    assert d["rows"][-1]["features"]["MeshVolume"] is None
    p = str(tmp_path / "s.json")
    save_shape(p, res)
    back = json.load(open(p))
    assert back["rows"][0]["features"] == res.rows[0].features
    assert back["rows"][0]["moments"]["N"] == res.rows[0].voxels
    c = str(tmp_path / "s.csv")
    save_shape(c, res)
    lines = open(c).read().splitlines()
    assert lines[0].split(",") == ["label", "name", "voxels"] + list(sh.SHAPE_FEATURES)
    assert len(lines) == 1 + len(res.rows) and lines[-1].endswith("nan")
    with pytest.raises(SystemExit):
        save_shape(str(tmp_path / "s.txt"), res)


def _host_inferer():
    from lungmask_b200.mask import LMInferer
    inf = object.__new__(LMInferer)
    inf.engine = types.SimpleNamespace(device=0, n_classes={0: 3})
    inf.modelname = "R231"
    return inf


def test_argument_errors():
    inf = _host_inferer()
    m = np.zeros((4, 5, 6), np.uint8)
    with pytest.raises(ValueError, match="spacing"):
        inf.shape(m)
    for bad in ((1.0, 1.0), (1.0, 0.0, 1.0), (1.0, float("nan"), 1.0)):
        with pytest.raises(ValueError, match="spacing"):
            inf.shape(m, spacing=bad)
    with pytest.raises(TypeError, match="uint8 or bool"):
        inf.shape(m.astype(np.float32), spacing=(1, 1, 1))
    with pytest.raises(ValueError, match="shape"):
        inf.shape(np.zeros((4, 5), np.uint8), spacing=(1, 1, 1))


def test_cli_checks_the_path_first(tmp_path):
    from lungmask_b200.__main__ import main
    inp = tmp_path / "v.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    with pytest.raises(SystemExit, match="unsupported shape output"):
        main([str(inp), str(tmp_path / "m.npy"), "--shape", str(tmp_path / "s.xlsx")])
