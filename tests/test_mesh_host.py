"""The numpy statement of the surface meshes (lungmask_b200.mesh.mesh_host): its numbering against a per-cube loop over the
table, closedness and orientation, area and volume against the shape features, the placement in patient space, the
writers and the argument checks.  CPU only."""
import itertools
import math
import struct

import numpy as np
import pytest

from lungmask_b200 import mesh as me
from lungmask_b200 import shape as sh

SPACING = (0.7, 0.8, 2.5)   # (x, y, z) mm


def loop_mesh(mask, row):
    """(index2, triangles) by a literal loop: every padded grid point in linear order and its three edges, then every
    cube in linear order and the triangles of its configuration."""
    member = (mask != 0) if row == 256 else (mask == row)
    n = member.shape

    def inside(q):
        return all(0 <= q[k] < n[k] for k in range(3)) and bool(member[tuple(q)])

    vid, index2 = {}, []
    for q in itertools.product(*[range(-1, n[k] + 1) for k in range(3)]):
        for m in range(3):
            r = list(q)
            r[m] += 1
            if r[m] <= n[m] and inside(q) != inside(r):
                vid[(q, m)] = len(index2)
                index2.append([2 * q[k] + (k == m) for k in range(3)])
    tris = []
    for p in itertools.product(*[range(-1, n[k]) for k in range(3)]):
        conf = sum(1 << k for k in range(8) if inside([p[j] + int(sh.CORNERS[k][j]) for j in range(3)]))
        for tri in sh.TRIANGLES[conf]:
            ids = []
            for e in tri:
                a, _, m = sh.EDGES[e]
                ids.append(vid[(tuple(p[j] + int(sh.CORNERS[a][j]) for j in range(3)), m)])
            tris.append(ids)
    return np.array(index2, np.int64).reshape(-1, 3), np.array(tris, np.int64).reshape(-1, 3)


def random_mask(seed, shape, labels):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, labels + 1, shape) * (rng.random(shape) < 0.7)).astype(np.uint8)


def rows_of(mask):
    return [int(x) for x in np.unique(mask) if x] + [256]


def check_closed(tris):
    """Every directed edge of the triangles is matched by its reverse exactly once."""
    t = np.asarray(tris, np.int64)
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    key = e[:, 0] * (int(t.max()) + 1) + e[:, 1]
    rev = e[:, 1] * (int(t.max()) + 1) + e[:, 0]
    assert len(np.unique(key)) == len(key), "a directed edge appears twice"
    assert np.array_equal(np.sort(key), np.sort(rev)), "a directed edge has no reverse"


@pytest.mark.parametrize("seed,shape,labels", [(0, (4, 5, 6), 1), (1, (5, 3, 7), 3), (2, (1, 6, 5), 2), (3, (6, 1, 4), 2),
                                               (4, (3, 5, 1), 3), (5, (1, 1, 7), 2), (6, (1, 1, 1), 1), (7, (6, 6, 6), 4)])
def test_against_loop(seed, shape, labels):
    m = random_mask(seed, shape, labels)
    m[0, 0, 0], m[-1, -1, -1] = 1, labels   # touch all six faces
    for row in rows_of(m):
        got = me.mesh_host(m, row, SPACING)
        index2, tris = loop_mesh(m, row)
        np.testing.assert_array_equal(got.index2, index2)
        np.testing.assert_array_equal(got.triangles, tris)
        assert got.index2.dtype == np.int32 and got.triangles.dtype == np.int32 and got.vertices.dtype == np.float64
        np.testing.assert_array_equal(got.vertices, index2[:, ::-1] * 0.5 * np.array(SPACING))


def test_full_and_empty():
    full = np.ones((3, 4, 5), np.uint8)
    got = me.mesh_host(full, 1, SPACING)
    index2, tris = loop_mesh(full, 1)
    np.testing.assert_array_equal(got.index2, index2)
    np.testing.assert_array_equal(got.triangles, tris)
    empty = me.mesh_host(np.zeros((3, 4, 5), np.uint8), 256, SPACING)
    assert empty.n_vertices == empty.n_triangles == 0 and empty.area() == empty.volume() == 0.0


@pytest.mark.parametrize("seed", range(4))
def test_closed_and_oriented(seed):
    m = random_mask(10 + seed, (7, 8, 9), 3)
    for row in rows_of(m):
        check_closed(me.mesh_host(m, row, SPACING).triangles)


def ball(r):
    z, y, x = np.ogrid[-r - 1:r + 2, -r - 1:r + 2, -r - 1:r + 2]
    return (x * x + y * y + z * z <= r * r).astype(np.uint8)


def shape_area_volume(mask, row, spacing):
    counts, possum, moments = sh.cube_sums_host(mask)
    f = sh.features(int(moments[row][0]), counts[row], possum[row], moments[row], np.zeros(4), spacing)
    return f["SurfaceArea"], f["MeshVolume"]


def boxes():
    m = np.zeros((6, 9, 11), np.uint8)
    m[1:4, 2:8, 3:10] = 1
    m[4:6, 0:9, 0:5] = 2   # touches the array's faces
    return m


@pytest.mark.parametrize("name", ["voxel", "boxes", "ball", "random"])
def test_area_volume_match_shape(name):
    one = np.zeros((3, 3, 3), np.uint8)
    one[1, 1, 1] = 1
    mask = {"voxel": one, "boxes": boxes(), "ball": ball(12), "random": random_mask(20, (9, 10, 11), 3)}[name]
    for row in rows_of(mask):
        A, V = shape_area_volume(mask, row, SPACING)
        got = me.mesh_host(mask, row, SPACING)
        assert math.isclose(got.area(), A, rel_tol=1e-12), (row, got.area(), A)
        assert math.isclose(got.volume(), V, rel_tol=1e-12), (row, got.volume(), V)
    if name == "voxel":   # the one-voxel octahedron
        got = me.mesh_host(mask, 1, (1.0, 1.0, 1.0))
        assert (got.n_vertices, got.n_triangles) == (6, 8)
        assert math.isclose(got.volume(), 1.0 / 6.0, rel_tol=1e-15)


def rotation(ax, ay, az):
    cx, sx, cy, sy, cz, sz = math.cos(ax), math.sin(ax), math.cos(ay), math.sin(ay), math.cos(az), math.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def test_rotation_and_reflection_keep_the_volume():
    mask = ball(12)
    mask[:, :, :14] *= 2
    origin = (-183.5, 97.25, -1204.0)
    for row in rows_of(mask):
        A, V = shape_area_volume(mask, row, SPACING)
        R = rotation(0.3, -0.7, 1.1)
        for D in (R, R @ np.diag([1.0, 1.0, -1.0]), np.diag([-1.0, 1.0, 1.0])):
            got = me.mesh_host(mask, row, SPACING, origin, D.ravel())
            assert V > 0 and got.volume() > 0
            assert math.isclose(got.volume(), V, rel_tol=1e-12), (row, np.linalg.det(D), got.volume(), V)
            assert math.isclose(got.area(), A, rel_tol=1e-12)
        plain = me.mesh_host(mask, row, SPACING, origin, R.ravel())
        flipped = me.mesh_host(mask, row, SPACING, origin, (R @ np.diag([1.0, 1.0, -1.0])).ravel())
        np.testing.assert_array_equal(flipped.triangles, plain.triangles[:, [0, 2, 1]])
        np.testing.assert_array_equal(flipped.index2, plain.index2)


def test_placement_statement():
    m = random_mask(30, (4, 5, 6), 2)
    D = rotation(0.2, 0.4, -0.9)
    o = (12.5, -30.25, 7.0)
    got = me.mesh_host(m, 256, SPACING, o, D.ravel())
    u = got.index2.astype(np.float64)
    want = np.empty_like(u)
    for i in range(len(u)):
        t = [SPACING[0] * (u[i, 2] * 0.5), SPACING[1] * (u[i, 1] * 0.5), SPACING[2] * (u[i, 0] * 0.5)]
        for c in range(3):
            want[i, c] = ((o[c] + D[c, 0] * t[0]) + D[c, 1] * t[1]) + D[c, 2] * t[2]
    assert got.vertices.view(np.uint64).tolist() == want.view(np.uint64).tolist()


def test_ras_flip_is_exact():
    m = random_mask(31, (5, 6, 7), 2)
    D = rotation(0.5, 0.1, 0.3).ravel()
    o = (-100.3, 55.1, 9.9)
    lps = me.mesh_host(m, 256, SPACING, o, D, "lps")
    ras = me.mesh_host(m, 256, SPACING, o, D, "ras")
    assert ras.space == "ras"
    np.testing.assert_array_equal(ras.triangles, lps.triangles)
    want = lps.vertices.copy()
    want[:, :2] = -want[:, :2]
    assert ras.vertices.view(np.uint64).tolist() == want.view(np.uint64).tolist()
    assert math.isclose(ras.volume(), lps.volume(), rel_tol=1e-12) and ras.volume() > 0


# ---- writers ----------------------------------------------------------------------------------------------------------
def read_stl(path):
    b = open(path, "rb").read()
    n = struct.unpack_from("<I", b, 80)[0]
    rec = np.frombuffer(b, np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("attr", "<u2")]), count=n, offset=84)
    assert len(b) == 84 + 50 * n and not b.startswith(b"solid")
    return rec["n"], rec["v"]


def read_obj(path):
    V, F = [], []
    for line in open(path):
        if line.startswith("v "):
            V.append([float(x) for x in line.split()[1:]])
        elif line.startswith("f "):
            F.append([int(x) - 1 for x in line.split()[1:]])
    return np.array(V).reshape(-1, 3), np.array(F, np.int64).reshape(-1, 3)


def read_ply(path):
    b = open(path, "rb").read()
    end = b.index(b"end_header\n") + len(b"end_header\n")
    head = b[:end].decode("ascii").splitlines()
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int([h for h in head if h.startswith("element vertex")][0].split()[-1])
    nf = int([h for h in head if h.startswith("element face")][0].split()[-1])
    V = np.frombuffer(b, "<f8", count=3 * nv, offset=end).reshape(-1, 3)
    F = np.frombuffer(b, np.dtype([("n", "u1"), ("i", "<i4", 3)]), count=nf, offset=end + 24 * nv)
    assert np.all(F["n"] == 3) and len(b) == end + 24 * nv + 13 * nf
    return V, F["i"].astype(np.int64)


def test_writers_round_trip(tmp_path):
    from lungmask_b200 import io as lio
    m = me.mesh_host(random_mask(40, (5, 6, 7), 2), 256, SPACING, (1.5, -2.25, 3.0), rotation(0.1, 0.2, 0.3).ravel())
    lio.save_mesh(str(tmp_path / "m.ply"), m)
    V, F = read_ply(str(tmp_path / "m.ply"))
    assert V.view(np.uint64).tolist() == m.vertices.view(np.uint64).tolist()
    np.testing.assert_array_equal(F, m.triangles)
    lio.save_mesh(str(tmp_path / "m.obj"), m)
    V, F = read_obj(str(tmp_path / "m.obj"))
    assert V.view(np.uint64).tolist() == m.vertices.view(np.uint64).tolist()   # %.17g round-trips a double
    np.testing.assert_array_equal(F, m.triangles)
    lio.save_mesh(str(tmp_path / "m.STL"), m)
    N, P = read_stl(str(tmp_path / "m.STL"))
    T = m.triangles
    np.testing.assert_array_equal(P, m.vertices[T].astype(np.float32))
    a, b, c = (m.vertices[T[:, k]] for k in range(3))
    n = np.cross(b - a, c - a)
    np.testing.assert_array_equal(N, (n / np.linalg.norm(n, axis=1)[:, None]).astype(np.float32))


def test_stl_degenerate_triangle_has_zero_normal(tmp_path):
    from lungmask_b200 import io as lio
    V = np.array([[0.0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0]])
    T = np.array([[0, 1, 2], [0, 1, 3]], np.int32)
    lio.save_mesh(str(tmp_path / "d.stl"), me.Mesh(1, "x", V, np.zeros((4, 3), np.int32), T))
    N, _ = read_stl(str(tmp_path / "d.stl"))
    np.testing.assert_array_equal(N, [[0, 0, 0], [0, 0, 1]])


def test_empty_mesh_writes(tmp_path):
    from lungmask_b200 import io as lio
    m = me.mesh_host(np.zeros((2, 2, 2), np.uint8), 1, SPACING)
    for ext in ("stl", "obj", "ply"):
        lio.save_mesh(str(tmp_path / ("e." + ext)), m)
    assert read_stl(str(tmp_path / "e.stl"))[1].shape == (0, 3, 3)
    assert read_ply(str(tmp_path / "e.ply"))[0].shape == (0, 3)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals(tmp_path):
    from lungmask_b200 import io as lio
    m = np.zeros((2, 3, 4), np.uint8)
    for kw, msg in (({"spacing": None}, "spacing"), ({"spacing": (1.0, 0.0, 1.0)}, "spacing"),
                    ({"spacing": (1.0, 1.0)}, "spacing"), ({"space": "xyz"}, "space"), ({"row": 0}, "row"),
                    ({"row": 257}, "row"), ({"row": "lungs"}, "row"), ({"row": True}, "row"),
                    ({"direction": (1.0, 0.0, 0.0)}, "direction"), ({"direction": np.zeros(9)}, "singular"),
                    ({"direction": (1.0, 0, 0, 0, 1, 0, 0, 0, float("nan"))}, "direction"),
                    ({"origin": (0.0, float("inf"), 0.0)}, "origin"), ({"origin": (0.0, 0.0)}, "origin")):
        args = {"mask": m, "row": 1, "spacing": SPACING}
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            me.mesh_host(**args)
    with pytest.raises(ValueError, match="mask"):
        me.mesh_host(np.zeros((3, 4), np.uint8), 1, SPACING)
    with pytest.raises(ValueError, match="twice"):
        me.check_rows([1, "lung", 256])
    with pytest.raises(ValueError, match="empty"):
        me.check_rows([])
    assert me.check_rows([3, "lung", 1]) == [3, 256, 1]
    me.check_counts(1, me.MAX_ELEMENTS, me.MAX_ELEMENTS)
    for nv, nt in ((me.MAX_ELEMENTS + 1, 0), (0, me.MAX_ELEMENTS + 1)):
        with pytest.raises(ValueError, match="2\\^31 - 1"):
            me.check_counts("lung", nv, nt)
    with pytest.raises(SystemExit, match="mesh output format"):
        lio.save_mesh(str(tmp_path / "m.vtk"), me.mesh_host(m, 1, SPACING))
    assert not (tmp_path / "m.vtk").exists()


def test_geometry_from_image():
    from lungmask_b200 import io as lio
    D = tuple(rotation(0.1, 0.0, 0.0).ravel())
    v = lio.Volume(np.zeros((2, 3, 4), np.int16), (0.5, 0.6, 2.0), (1.0, 2.0, 3.0), D)
    sp, o, d = me.geometry(image=v)
    assert sp == (0.5, 0.6, 2.0) and o == (1.0, 2.0, 3.0) and np.array_equal(np.ravel(d), D)
    assert me.geometry(spacing=(1.0, 1.0, 1.0), image=v)[0] == (1.0, 1.0, 1.0)
    assert me.geometry(spacing=(1.0, 2.0, 3.0))[1:] == ((0.0, 0.0, 0.0), ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)))
    with pytest.raises(ValueError, match="spacing"):
        me.geometry()


def test_table_codes():
    """The codes the device reads name the table's edges: (corner a << 2) | axis m with a the lower corner."""
    assert me.TABLE_OFFSETS[0] == 0 and me.TABLE_OFFSETS[-1] * 3 == len(me.TABLE_CODES)
    for c in range(256):
        for t, tri in enumerate(sh.TRIANGLES[c]):
            for k, e in enumerate(tri):
                code = int(me.TABLE_CODES[(me.TABLE_OFFSETS[c] + t) * 3 + k])
                a, b, m = sh.EDGES[e]
                assert (code >> 2, code & 3) == (a, m) and b == a | (4 >> m)
                assert ((c >> a) & 1) != ((c >> b) & 1)


def test_cli_flags_and_checks_before_segmentation(tmp_path):
    from lungmask_b200.__main__ import build_parser, main, mesh_file_name
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    a = build_parser().parse_args([str(inp), "out.npy"])
    assert (a.mesh, a.mesh_format, a.mesh_space) == (None, "stl", "lps")
    a = build_parser().parse_args([str(inp), "out.npy", "--mesh", "d", "--mesh-format", "ply", "--mesh-space", "ras"])
    assert (a.mesh, a.mesh_format, a.mesh_space) == ("d", "ply", "ras")
    for flag, value in (("--mesh-format", "vtk"), ("--mesh-space", "xyz")):
        with pytest.raises(SystemExit):
            build_parser().parse_args([str(inp), "out.npy", "--mesh", "d", flag, value])
    out = str(tmp_path / "m.npy")
    (tmp_path / "file").write_text("")
    # every check ends the run before the volume is segmented (that would need a model and a GPU)
    for path, msg in ((str(tmp_path / "file"), "not a directory"), (str(tmp_path / "no" / "such"), "parent directory")):
        with pytest.raises(SystemExit, match=msg):
            main([str(inp), out, "--mesh", path])
    assert mesh_file_name(me.Mesh(1, "right lung", None, None, None), "stl") == "right_lung.stl"
    assert mesh_file_name(me.Mesh(1, "left upper lobe", None, None, None), "obj") == "left_upper_lobe.obj"
    assert mesh_file_name(me.Mesh("lung", "lung", None, None, None), "ply") == "lung.ply"
    assert mesh_file_name(me.Mesh(7, "label 7", None, None, None), "stl") == "label_7.stl"
