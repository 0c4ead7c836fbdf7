"""The host statement of LMInferer.resample (lungmask_b200.resample; DESIGN §4.19), without a GPU: the output grid
against a literal per-axis transcription of PyRadiomics' resampleImage, the B-spline decomposition against a scalar
per-line loop bit for bit, the interpolant against scipy.ndimage.map_coordinates(order=3, mode="mirror"), the nearest
and outside rules against literal loops, the output casts, the refusals, and the CLI checks of --resample."""
import math

import numpy as np
import pytest

from lungmask_b200 import resample as rsm


# ---- grid --------------------------------------------------------------------------------------------------------------

def grid_literal(shape, ms, rs, lo, size, pad):
    """PyRadiomics' resampleImage grid, one axis at a time in Python floats -> (crop, spacing, start, tables)."""
    N = shape[::-1]
    rs = [ms[d] if rs[d] == 0 else rs[d] for d in range(3)]
    rs = [ms[d] if size[d] == 1 else rs[d] for d in range(3)]
    if all(abs(ms[d] - rs[d]) <= 1e-8 + 1e-5 * abs(rs[d]) for d in range(3)):
        L = [max(lo[d] - pad, 0) for d in range(3)]
        U = [min(lo[d] + size[d] - 1 + pad, N[d] - 1) for d in range(3)]
        return True, list(ms), [float(x) for x in L], [[float(L[d] + k) for k in range(U[d] - L[d] + 1)] for d in range(3)]
    start, tables = [], []
    for d in range(3):
        r = ms[d] / rs[d]
        L = max(math.floor((lo[d] - 0.5) * r - pad), 0)
        U = min(math.ceil((lo[d] + size[d] - 0.5) * r + pad), math.ceil(N[d] * r) - 1)
        s = 0.5 * (rs[d] - ms[d]) / ms[d] + L / r
        start.append(s)
        tables.append([s + k * (rs[d] / ms[d]) for k in range(U - L + 1)])
    return False, rs, start, tables


def _box_mask(shape, lo, size):
    m = np.zeros(shape, np.uint8)
    m[lo[2]:lo[2] + size[2], lo[1]:lo[1] + size[1], lo[0]:lo[0] + size[0]] = 1
    return m


GRID_CASES = [
    # shape (z, y, x), ms, rs, lo (x, y, z), size (x, y, z), pad
    ((40, 60, 60), (0.7, 0.7, 1.25), (1.0, 1.0, 1.0), (10, 12, 5), (30, 20, 20), 5),       # down in-plane, up in z
    ((20, 30, 30), (1.5, 1.5, 2.5), (0.5, 0.5, 0.5), (4, 6, 3), (10, 12, 8), 2),           # upsampling
    ((20, 30, 30), (0.5, 0.5, 0.5), (2.0, 2.0, 2.0), (3, 3, 3), (20, 20, 10), 5),          # downsampling
    ((20, 30, 30), (0.7, 0.8, 2.5), (1.0, 0.0, 1.0), (2, 5, 4), (20, 10, 9), 3),           # a 0 entry keeps y
    ((20, 30, 30), (0.7, 0.7, 2.5), (1.0, 1.0, 1.0), (2, 5, 7), (20, 10, 1), 3),           # a one-slice box keeps z
    ((12, 17, 19), (0.9, 1.1, 3.0), (1.0, 1.0, 1.0), (0, 0, 0), (19, 17, 12), 5),          # touches every face
    ((12, 17, 19), (0.9, 1.1, 3.0), (0.6, 0.6, 1.3), (0, 0, 0), (19, 17, 12), 0),          # pad 0, every face
    ((12, 17, 19), (0.9, 1.1, 3.0), (1.0, 1.0, 1.0), (3, 2, 1), (5, 6, 4), 0),             # pad 0
    ((12, 17, 19), (1.0, 1.0, 2.0), (1.000001, 1.0, 2.0), (3, 2, 1), (5, 6, 4), 2),        # allclose: crop only
    ((12, 17, 19), (1.0, 1.0, 2.0), (0.0, 0.0, 0.0), (0, 0, 0), (19, 17, 12), 4),          # all 0: crop only, clamped
]


@pytest.mark.parametrize("shape,ms,rs,lo,size,pad", GRID_CASES)
def test_grid_matches_literal(shape, ms, rs, lo, size, pad):
    crop, spacing, start, tables = grid_literal(shape, ms, rs, lo, size, pad)
    g = rsm.grid(shape, ms, rs, lo, size, pad)
    assert g.crop == crop
    assert list(g.spacing) == list(spacing)
    assert list(g.start) == list(start)
    assert g.size == tuple(len(t) for t in tables)
    assert g.shape == tuple(len(t) for t in tables[::-1])
    for got, want in zip(g.tables, tables):
        assert got.dtype == np.float64
        assert np.array_equal(got, np.array(want))
    assert (rsm.bounding_box(_box_mask(shape, lo, size))) == (tuple(lo), tuple(size))


def test_grid_clamps_act():
    # a box touching every face with a pad: both the lower clamp (0) and the upper clamp (ceil(N r) - 1) decide
    g = rsm.grid((12, 17, 19), (0.9, 1.1, 3.0), (1.0, 1.0, 1.0), (0, 0, 0), (19, 17, 12), 5)
    for d, n in enumerate((19, 17, 12)):
        r = (0.9, 1.1, 3.0)[d] / 1.0
        assert g.tables[d][0] == 0.5 * (1.0 - (0.9, 1.1, 3.0)[d]) / (0.9, 1.1, 3.0)[d]
        assert g.size[d] == math.ceil(n * r)


def test_new_origin():
    D = (0.0, 1.0, 0.0, -1.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    got = rsm.new_origin((10.0, 20.0, 30.0), D, (0.5, 0.7, 2.0), (1.0, 2.0, -0.25))
    want = np.array([10.0, 20.0, 30.0]) + np.array(D).reshape(3, 3) @ (np.array([0.5, 0.7, 2.0]) * np.array([1.0, 2.0, -0.25]))
    assert got == tuple(want)


# ---- decomposition -----------------------------------------------------------------------------------------------------

def decompose_line(values):
    """The statement's 1-D decomposition of one line, scalar Python floats."""
    c = [float(v) for v in values]
    N = len(c)
    if N == 1:
        return c
    z = math.sqrt(3.0) - 2.0
    lam = (1.0 - z) * (1.0 - 1.0 / z)
    c = [v * lam for v in c]
    if N >= 19:
        s, zn = c[0], z
        for n in range(1, 18):
            s = s + zn * c[n]
            zn = zn * z
    else:
        zn, iz, z2n = z, 1.0 / z, z
        for _ in range(N - 2):
            z2n = z2n * z
        s = c[0] + z2n * c[N - 1]
        z2n = z2n * (z2n * iz)
        for n in range(1, N - 1):
            s = s + (zn + z2n) * c[n]
            zn = zn * z
            z2n = z2n * iz
        s = s / (1.0 - zn * zn)
    c[0] = s
    for n in range(1, N):
        c[n] = c[n] + z * c[n - 1]
    c[N - 1] = (z / (z * z - 1.0)) * (z * c[N - 2] + c[N - 1])
    for n in range(N - 2, -1, -1):
        c[n] = z * (c[n + 1] - c[n])
    return c


def decompose_literal(vol):
    c = vol.astype(np.float64)
    for axis in (2, 1, 0):
        moved = np.moveaxis(c, axis, -1)
        out = np.empty_like(moved)
        for idx in np.ndindex(moved.shape[:-1]):
            out[idx] = decompose_line(moved[idx])
        c = np.moveaxis(out, -1, axis)
    return c


def _u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("n", [1, 2, 3, 17, 18, 19, 64])
def test_decomposition_bit_exact(n):
    rng = np.random.default_rng(n)
    for shape in ((n, 3, 2), (2, n, 3), (3, 2, n)):
        vol = rng.integers(-1024, 1500, size=shape).astype(np.int16)
        assert np.array_equal(_u64(rsm.decompose_host(vol)), _u64(decompose_literal(vol)))
    f = rng.normal(0, 300, size=(2, 3, n))
    assert np.array_equal(_u64(rsm.decompose_host(f)), _u64(decompose_literal(f)))


# ---- evaluation --------------------------------------------------------------------------------------------------------

def _points(n, k, rng):
    """k continuous indices inside [-0.5, n - 0.5), including the two edge bands."""
    c = rng.uniform(-0.5, n - 0.5, size=k)
    c[0], c[1] = -0.5, np.nextafter(n - 0.5, -1.0)
    c[2] = rng.uniform(-0.5, 0.0)
    c[3] = rng.uniform(n - 1, n - 0.5) if n > 1 else rng.uniform(0.0, 0.5)
    return c


@pytest.mark.parametrize("shape", [(19, 23, 40), (3, 18, 25), (2, 5, 64), (1, 7, 30), (4, 1, 2)])
def test_interpolant_matches_scipy(shape):
    from scipy import ndimage
    rng = np.random.default_rng(sum(shape))
    vol = rng.integers(-1024, 1500, size=shape).astype(np.int16)
    tables = tuple(_points(n, 9, rng) for n in shape[::-1])
    got = rsm._bspline_planes(rsm.decompose_host(vol), tables, np.arange(len(tables[2])))
    zz, yy, xx = np.meshgrid(tables[2], tables[1], tables[0], indexing="ij")
    want = ndimage.map_coordinates(vol.astype(np.float64), [zz.ravel(), yy.ravel(), xx.ravel()], order=3,
                                   mode="mirror").reshape(got.shape)
    assert np.max(np.abs(got - want)) <= 1e-9 * np.max(np.abs(vol))


def test_separable_sum_equals_per_voxel_order():
    """_bspline_planes forms every voxel's 64-tap sum in the order of the device (x innermost, then y, then z)."""
    rng = np.random.default_rng(7)
    vol = rng.normal(0, 100, size=(5, 6, 7))
    coeff = rsm.decompose_host(vol)
    tables = tuple(_points(n, 5, rng) for n in vol.shape[::-1])
    got = rsm._bspline_planes(coeff, tables, np.arange(5))
    (ix, wx), (iy, wy), (iz, wz) = (rsm.bspline_weights(t) for t in tables)
    ix, iy, iz = rsm.mirror(ix, 7), rsm.mirror(iy, 6), rsm.mirror(iz, 5)
    for kz in range(5):
        for ky in range(5):
            for kx in range(5):
                v = 0.0
                for a in range(4):
                    sy = 0.0
                    for b in range(4):
                        sx = 0.0
                        for c in range(4):
                            sx = sx + float(wx[kx, c]) * float(coeff[iz[kz, a], iy[ky, b], ix[kx, c]])
                        sy = sy + float(wy[ky, b]) * sx
                    v = v + float(wz[kz, a]) * sy
                assert got[kz, ky, kx] == v


def test_mirror_and_weights():
    assert list(rsm.mirror(np.arange(-2, 4), 2)) == [0, 1, 0, 1, 0, 1]
    assert list(rsm.mirror(np.arange(-2, 7), 5)) == [2, 1, 0, 1, 2, 3, 4, 3, 2]
    assert list(rsm.mirror(np.arange(-2, 3), 1)) == [0] * 5
    _, w = rsm.bspline_weights(np.array([0.0, 0.25, 3.5]))
    assert np.allclose(w.sum(axis=1), 1.0)
    assert np.allclose(w[0], [1 / 6, 4 / 6, 1 / 6, 0])


def _nearest_literal(arr, tables):
    n0, n1, n2 = arr.shape
    out = np.zeros((len(tables[2]), len(tables[1]), len(tables[0])), arr.dtype)
    for kz, z in enumerate(tables[2]):
        for ky, y in enumerate(tables[1]):
            for kx, x in enumerate(tables[0]):
                if not (-0.5 <= z < n0 - 0.5 and -0.5 <= y < n1 - 0.5 and -0.5 <= x < n2 - 0.5):
                    continue
                i = [min(max(math.floor(c + 0.5), 0), n - 1) for c, n in ((z, n0), (y, n1), (x, n2))]
                out[kz, ky, kx] = arr[i[0], i[1], i[2]]
    return out


@pytest.mark.parametrize("interpolator", ["bspline", "nearest"])
def test_points_outside_nearest_and_mask(interpolator):
    rng = np.random.default_rng(3)
    vol = rng.integers(-1000, 1000, size=(6, 9, 11)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    mask[1:5, 2:8, 1:10] = rng.integers(1, 4, size=(4, 6, 9))
    # upsampling with a pad reaching past every face: the edge samples fall outside the buffer
    img, m, g = rsm.resample_host(vol, mask, (1.0, 1.0, 2.0), (0.45, 0.45, 0.7), interpolator, pad_distance=3)
    shape = vol.shape
    outside = ~(rsm.inside(g.tables[2], shape[0])[:, None, None] & rsm.inside(g.tables[1], shape[1])[None, :, None]
                & rsm.inside(g.tables[0], shape[2])[None, None, :])
    assert outside.any()
    assert not img[outside].any() and not m[outside].any()
    assert np.array_equal(m, _nearest_literal(mask, g.tables))
    if interpolator == "nearest":
        assert np.array_equal(img, _nearest_literal(vol, g.tables))


def test_crop_only_keeps_values():
    rng = np.random.default_rng(5)
    vol = rng.normal(0, 100, size=(8, 9, 10)).astype(np.float32)
    mask = np.zeros(vol.shape, np.uint8)
    mask[2:5, 3:6, 1:4] = 2
    img, m, g = rsm.resample_host(vol, mask, (0.8, 0.8, 2.0), (0.8, 0.8, 2.0), "bspline", pad_distance=1)
    assert g.crop and g.start == (0.0, 2.0, 1.0)
    assert np.array_equal(img, vol[1:6, 2:7, 0:5]) and np.array_equal(m, mask[1:6, 2:7, 0:5])


# ---- casts -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.uint8, np.int8, np.int16, np.int32, np.int64, np.uint16, np.uint32])
def test_integer_casts(dtype):
    info = np.iinfo(dtype)
    lo, hi = float(info.min), float(info.max)
    v = np.array([-1e30, lo - 0.5, lo + 0.7, -1.9, -0.5, -0.0, 0.5, 1.9, 2.5, hi - 0.3, hi + 0.5, 1e30])
    got = rsm.cast_host(v, dtype)
    assert got.dtype == dtype
    want = []
    for x in v:
        x = min(max(x, lo), rsm.int_bounds(dtype)[1])
        want.append(int(math.trunc(x)))
    assert [int(x) for x in got] == want
    assert int(got[0]) == info.min
    assert int(got[-1]) == (info.max if dtype != np.int64 else 2 ** 63 - 1024)


def test_float_casts():
    v = np.array([1.0 + 2.0 ** -30, -3.000000476837158, 1234.5678, 0.1])
    assert np.array_equal(rsm.cast_host(v, np.float32), v.astype(np.float32))
    assert rsm.cast_host(v, np.float32)[0] == np.float32(1.0)
    assert np.array_equal(rsm.cast_host(v, np.float16), v.astype(np.float16))
    assert rsm.cast_host(v, np.float64) is not v and np.array_equal(rsm.cast_host(v, np.float64), v)


def test_int16_bspline_round_trip_dtype():
    rng = np.random.default_rng(11)
    vol = rng.integers(-1024, 1500, size=(6, 10, 12)).astype(np.int16)
    mask = np.ones(vol.shape, np.uint8)
    img, m, g = rsm.resample_host(vol, mask, (0.7, 0.7, 1.5), (1.0, 1.0, 1.0))
    assert img.dtype == np.int16 and m.dtype == np.uint8
    f, _, _ = rsm.resample_host(vol.astype(np.float64), mask, (0.7, 0.7, 1.5), (1.0, 1.0, 1.0))
    assert np.array_equal(img, np.trunc(np.clip(f, -32768, 32767)).astype(np.int16))


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refusals():
    vol = np.zeros((4, 5, 6), np.float32)
    mask = np.ones(vol.shape, np.uint8)
    for bad in (np.nan, np.inf, -np.inf):
        v = vol.copy()
        v[1, 2, 3] = bad
        with pytest.raises(ValueError, match="NaN"):
            rsm.resample_host(v, mask, (1, 1, 1))
    with pytest.raises(ValueError, match="empty"):
        rsm.resample_host(vol, np.zeros_like(mask), (1, 1, 1))
    with pytest.raises(ValueError, match="shape"):
        rsm.resample_host(vol, mask[:, :, :5], (1, 1, 1))
    for sp in ((1, 1), (1, 0, 1), (1, -1, 1), (1, np.nan, 1), None, "abc"):
        with pytest.raises(ValueError, match="spacing"):
            rsm.resample_host(vol, mask, sp)
    for rs in ((1, -1, 1), (1, np.inf, 1), (1, 1)):
        with pytest.raises(ValueError, match="resampled_spacing"):
            rsm.resample_host(vol, mask, (1, 1, 1), rs)
    for pad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="pad_distance"):
            rsm.resample_host(vol, mask, (1, 1, 1), (2, 2, 2), pad_distance=pad)
    with pytest.raises(ValueError, match="interpolator"):
        rsm.resample_host(vol, mask, (1, 1, 1), interpolator="linear")
    with pytest.raises(TypeError, match="bool"):
        rsm.resample_host(vol.astype(bool), mask, (1, 1, 1))
    with pytest.raises(ValueError, match="2\\^32"):
        rsm.check_shape((1 << 11, 1 << 11, 1 << 10))
    with pytest.raises(ValueError, match="2\\^32"):
        rsm.grid((100, 100, 100), (1.0, 1.0, 1.0), (0.001, 0.001, 0.001), (0, 0, 0), (100, 100, 100), 0)
    assert rsm.parse_spacing("1, 1,0.5") == (1.0, 1.0, 0.5)
    for spec in ("1,1", "a,b,c", "1,1,-1", "1,1,1,1"):
        with pytest.raises(ValueError):
            rsm.parse_spacing(spec)


def test_abi_refuses_null_arguments():
    from lungmask_b200 import _native
    L = _native.lib()
    p = None
    assert L.lm_bspline_coefficients_dev(None, p, 0, 1, 1, 1, p, None) == -1
    assert "NULL" in L.lm_last_error().decode()
    assert L.lm_resample_dev(None, p, 0, p, p, 1, 1, 1, p, p, p, 1, 1, 1, 0, p, p, None) == -1
    assert "NULL" in L.lm_last_error().decode()


# ---- CLI ---------------------------------------------------------------------------------------------------------------

def _cli_main(tmp_path, monkeypatch, argv):
    import lungmask_b200.__main__ as cli

    def no_load(*a, **k):
        raise AssertionError("the input was read before the arguments were checked")
    monkeypatch.setattr(cli, "load_input_image", no_load)
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    cli.main([str(src), str(tmp_path / "out.nii")] + argv)


@pytest.mark.parametrize("argv,msg", [
    (["--texture", "t.json", "--resample", "1,1"], "--resample"),
    (["--texture", "t.json", "--resample", "1,x,1"], "--resample"),
    (["--shape", "s.json", "--resample", "1,-1,1"], "--resample"),
    (["--statistics", "s.json", "--resample", "1,1,1"], "--resample: applies to"),
    (["--texture", "t.json", "--resample-interpolator", "nearest"], "--resample-interpolator"),
])
def test_cli_refusals_before_segmentation(tmp_path, monkeypatch, argv, msg):
    argv = [str(tmp_path / a) if a.endswith(".json") else a for a in argv]
    with pytest.raises(SystemExit, match=msg):
        _cli_main(tmp_path, monkeypatch, argv)


def test_cli_parser_refuses_unknown_interpolator(tmp_path):
    from lungmask_b200.__main__ import build_parser
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    with pytest.raises(SystemExit):
        build_parser().parse_args([str(src), "out.nii", "--resample", "1,1,1", "--resample-interpolator", "linear"])


def test_cli_resample_arguments(tmp_path):
    from lungmask_b200.__main__ import build_parser, resample_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    args = build_parser().parse_args([str(src), "out.nii", "--texture", "t.json", "--resample", "1,0,2.5"])
    assert resample_arguments(args) == ((1.0, 0.0, 2.5), "bspline")
    args = build_parser().parse_args([str(src), "out.nii", "--filtered", "f.json", "--resample", "1,1,1",
                                      "--resample-interpolator", "nearest"])
    assert resample_arguments(args) == ((1.0, 1.0, 1.0), "nearest")
    assert resample_arguments(build_parser().parse_args([str(src), "out.nii"])) is None
