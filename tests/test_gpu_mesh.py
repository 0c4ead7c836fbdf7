"""Surface meshes on the GPU (LMInferer.mesh, lm_mesh_counts_dev, lm_mesh_emit_dev) against the numpy statement
lungmask_b200.mesh.mesh_host: vertex numbering, doubled coordinates and triangles equal, positions bit-identical; area
and volume against LMInferer.shape; the CLI's files against the call."""
import math
import os

import numpy as np
import pytest

from lungmask_b200 import mesh as me
from oracle import synth

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 2.5)             # (x, y, z) mm; not dyadic
ORIGIN = (-183.7, 97.3, -1204.1)


def rotation(ax, ay, az):
    cx, sx, cy, sy, cz, sz = math.cos(ax), math.sin(ax), math.cos(ay), math.sin(ay), math.cos(az), math.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


ROTATED = rotation(0.3, -0.7, 1.1)
REFLECTED = ROTATED @ np.diag([1.0, 1.0, -1.0])


@pytest.fixture(scope="module")
def inf():
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


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def assert_same(got, want, what=""):
    got = got.numpy()
    np.testing.assert_array_equal(got.index2, want.index2, err_msg="index2 %s" % what)
    np.testing.assert_array_equal(got.triangles, want.triangles, err_msg="triangles %s" % what)
    np.testing.assert_array_equal(_bits(got.vertices), _bits(want.vertices), err_msg="vertices %s" % what)
    assert got.index2.dtype == np.int32 and got.triangles.dtype == np.int32


def check_exact(inf, mask, spacing=SPACING, origin=None, direction=None, space="lps"):
    """Every present row and "lung" of the CUDA-tensor call against mesh_host."""
    import torch
    m8 = np.ascontiguousarray(mask).view(np.uint8) if mask.dtype == bool else mask
    tm = _cuda(m8)
    rows = [int(x) for x in np.unique(m8) if x] + ["lung"]
    from lungmask_b200 import io as lio
    image = None
    if origin is not None:
        image = lio.Volume(np.zeros(m8.shape, np.int16), spacing, origin, tuple(np.ravel(direction)))
    res = inf.mesh(tm, spacing=None if image else spacing, image=image, rows=rows, space=space)
    assert [r.label for r in res.rows] == rows
    for got, r in zip(res.rows, rows):
        assert isinstance(got.vertices, torch.Tensor) and got.vertices.device == tm.device
        want = me.mesh_host(m8, r, spacing, origin, None if direction is None else np.ravel(direction), space)
        assert_same(got, want, "row %s" % r)
    return res


def random_labels(seed, shape, labels):
    import scipy.ndimage as ndi
    rng = np.random.default_rng(seed)
    field = ndi.gaussian_filter(rng.standard_normal(shape), 1.5)
    m = (field > np.quantile(field, 0.4)).astype(np.uint8)
    region = ndi.gaussian_filter(rng.standard_normal(shape), 2.5)
    cuts = np.quantile(region, np.linspace(0, 1, labels + 1)[1:-1])
    return m * (np.searchsorted(cuts, region) + 1).astype(np.uint8)


@pytest.mark.parametrize("seed,shape,labels", [(0, (13, 27, 35), 1), (1, (20, 33, 47), 3), (2, (5, 64, 17), 6),
                                               (3, (31, 16, 32), 2), (4, (24, 40, 64), 5), (5, (9, 70, 97), 4)])
def test_random_masks(inf, seed, shape, labels):
    check_exact(inf, random_labels(seed, shape, labels))


def test_geometry_and_spaces(inf):
    m = random_labels(10, (17, 29, 41), 3)
    for D in (ROTATED, REFLECTED):
        for space in ("lps", "ras"):
            res = check_exact(inf, m, SPACING, ORIGIN, D, space)
            assert res["lung"].numpy().volume() > 0


def test_speckle_full_empty(inf):
    rng = np.random.default_rng(11)
    check_exact(inf, rng.integers(0, 4, (11, 19, 37)).astype(np.uint8))          # speckle touching all six faces
    check_exact(inf, (rng.random((16, 33, 65)) < 0.5).astype(np.uint8))
    check_exact(inf, np.ones((11, 19, 37), np.uint8))
    res = inf.mesh(_cuda(np.zeros((6, 17, 33), np.uint8)), spacing=SPACING)
    assert [r.label for r in res.rows] == [1, 2, "lung"]
    assert all(r.n_vertices == r.n_triangles == 0 for r in res.rows)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 9, 10), (8, 1, 7), (6, 5, 1), (1, 1, 40), (1, 33, 1), (7, 8, 31),
                                   (8, 7, 32), (3, 4, 33)])
def test_extents(inf, shape):
    rng = np.random.default_rng(sum(shape))
    m = rng.integers(0, 3, shape).astype(np.uint8)
    m.reshape(-1)[0] = 1
    check_exact(inf, m)


def test_forty_labels(inf):
    rng = np.random.default_rng(6)
    m = np.zeros((18, 42, 50), np.uint8)
    for l in range(1, 41):
        z, y, x = rng.integers(0, 14), rng.integers(0, 36), rng.integers(0, 44)
        m[z:z + rng.integers(1, 5), y:y + rng.integers(1, 7), x:x + rng.integers(1, 7)] = l
    assert len(np.unique(m)) == 41
    check_exact(inf, m)


def test_input_paths_and_area_volume(inf):
    import torch
    from lungmask_b200 import io as lio
    m = random_labels(8, (14, 38, 29), 3)
    image = lio.Volume(np.zeros(m.shape, np.int16), SPACING, ORIGIN, tuple(REFLECTED.ravel()))
    tm = _cuda(m)
    before = tm.clone()
    a = inf.mesh(tm, image=image)
    assert torch.equal(tm, before), "the CUDA mask was modified"
    b = inf.mesh(m, image=image)
    c = inf.mesh(torch.from_numpy(m), image=image)
    d = inf.mesh(m > 0, image=image, rows=["lung"])
    assert [r.label for r in a.rows] == [r.label for r in b.rows] == [1, 2, 3, "lung"]
    assert [r.name for r in a.rows] == [r.name for r in b.rows]
    for ra, rb, rc in zip(a.rows, b.rows, c.rows):
        assert isinstance(rb.vertices, np.ndarray) and isinstance(rc.vertices, np.ndarray)
        assert_same(ra, rb)
        assert_same(ra, rc)
    assert_same(a["lung"], d["lung"].numpy())
    sf = inf.shape(m, spacing=SPACING)
    for r in b.rows:
        assert math.isclose(r.area(), sf[r.label]["SurfaceArea"], rel_tol=1e-12)
        assert math.isclose(r.volume(), sf[r.label]["MeshVolume"], rel_tol=1e-12)


def test_errors(inf):
    from lungmask_b200 import _native
    m = np.zeros((4, 5, 6), np.uint8)
    m[1:3, 1:4, 2:5] = 1
    for kw, msg in (({}, "spacing"), ({"spacing": SPACING, "space": "lpi"}, "space"),
                    ({"spacing": SPACING, "rows": [0]}, "row"), ({"spacing": SPACING, "rows": [1, 1]}, "twice")):
        with pytest.raises(ValueError, match=msg):
            inf.mesh(m, **kw)
    tm = _cuda(m)
    off, codes = me.TABLE_OFFSETS, me.TABLE_CODES
    geo = me.geometry_vector(SPACING, (0.0, 0.0, 0.0), ((1.0, 0, 0), (0, 1.0, 0), (0, 0, 1.0)))
    nv, nt = inf.engine.mesh_counts_dev(tm.data_ptr(), m.shape, 1, off, codes)
    assert (nv, nt) == (me.mesh_host(m, 1, SPACING).n_vertices, me.mesh_host(m, 1, SPACING).n_triangles)
    with pytest.raises(_native.NativeError, match="row"):
        inf.engine.mesh_counts_dev(tm.data_ptr(), m.shape, 0, off, codes)
    bad = codes.copy()
    bad[0] ^= 1 << 2   # another corner: the edge no longer crosses in its configuration, or is no edge
    with pytest.raises(_native.NativeError, match="configuration"):
        inf.engine.mesh_counts_dev(tm.data_ptr(), m.shape, 1, off, bad)
    import torch
    i2, v, t = (torch.empty((n, 3), dtype=dt, device="cuda:0") for n, dt in ((nv, torch.int32), (nv, torch.float64),
                                                                            (nt, torch.int32)))
    ptrs = (i2.data_ptr(), v.data_ptr(), t.data_ptr())
    with pytest.raises(_native.NativeError, match="counts"):
        inf.engine.mesh_emit_dev(tm.data_ptr(), m.shape, 1, off, codes, geo, nv, nt + 1, *ptrs)
    sing = geo.copy()
    sing[3:12] = 0.0
    with pytest.raises(_native.NativeError, match="singular"):
        inf.engine.mesh_emit_dev(tm.data_ptr(), m.shape, 1, off, codes, sing, nv, nt, *ptrs)
    with pytest.raises(_native.NativeError, match="2\\^31"):
        inf.engine.mesh_emit_dev(tm.data_ptr(), m.shape, 1, off, codes, geo, 2 ** 31, nt, *ptrs)
    inf.engine.mesh_emit_dev(tm.data_ptr(), m.shape, 1, off, codes, geo, nv, nt, *ptrs)
    want = me.mesh_host(m, 1, SPACING)
    np.testing.assert_array_equal(t.cpu().numpy(), want.triangles)


def five_lobes(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    lobes = m.copy()
    lobes[(m == 1) & (z >= S // 2)] = 2
    lobes[(m == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(m == 2) & (z < S // 2)] = 4
    lobes[(m == 2) & (z >= S // 2)] = 5
    return m, lobes


def test_full_size(inf):
    """300x512x512: the two-lung phantom and its five-lobe split, every row bit for bit; the "lung" row is closed."""
    from test_mesh_host import check_closed
    lungs, lobes = five_lobes(300, 512, 512)
    for m in (lungs, lobes):
        res = check_exact(inf, m, (0.703125, 0.703125, 1.25), ORIGIN, ROTATED)
    check_closed(res["lung"].triangles.cpu().numpy())


def test_cli(tmp_path):
    import torch
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    from test_mesh_host import read_obj
    wpath = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=48, head_gain=0.3), wpath)
    vol = synth.phantom(6, 160, 176, seed=24)
    src = lio.Volume(vol, (0.75, 0.5, 1.5), (10.0, -20.0, 30.0), tuple(ROTATED.ravel()))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = tmp_path / "meshes"
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", wpath, "--noprogress", "--batchsize", "4", "--mesh", str(out),
          "--mesh-format", "obj", "--mesh-space", "ras"])
    inf = LMInferer(modelpath=wpath, tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.mesh(inf.apply(v), image=v, space="ras")
    written = sorted(os.listdir(out))
    expect = sorted("%s.obj" % r.name.replace(" ", "_") for r in want.rows if r.n_triangles or r.label == "lung")
    assert written == expect and "lung.obj" in written
    for r in want.rows:
        name = "%s.obj" % r.name.replace(" ", "_")
        if name in written:
            V, F = read_obj(str(out / name))
            np.testing.assert_array_equal(_bits(V), _bits(r.vertices))
            np.testing.assert_array_equal(F, r.triangles)
