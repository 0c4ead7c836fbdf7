"""Voxel-based GLSZM, GLRLM, GLDM and NGTDM maps on the GPU (LMInferer.texture_maps, lm_texture_maps_dev): every map bit
for bit (uint64 patterns) against the numpy statement texture_maps.maps_host."""
import numpy as np
import pytest

from lungmask_b200 import first_order_maps as fm
from lungmask_b200 import texture as tx
from lungmask_b200 import texture_maps as tm
from oracle import synth

pytestmark = pytest.mark.gpu


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


def two_lungs(S, H, W, z0=0, z1=None):
    """The two-ellipsoid mask of an (S, H, W) volume, slices z0..z1."""
    z1 = S if z1 is None else z1
    z, y, x = np.ogrid[z0:z1, :H, :W]
    m = np.zeros((z1 - z0, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


def assert_bits(got, want, where=""):
    """Every plane of two TextureMaps equal as uint64 patterns."""
    assert list(got.maps) == list(want.maps)
    assert (got.low, got.n_levels, got.voxels, got.classes, got.gldm_alpha) == \
        (want.low, want.n_levels, want.voxels, want.classes, want.gldm_alpha), where
    for k, m in got.maps.items():
        g = np.ascontiguousarray(m.cpu().numpy() if hasattr(m, "cpu") else m)
        w = want.maps[k]
        bad = g.view(np.uint64) != w.view(np.uint64)
        assert not bad.any(), (where, k, int(bad.sum()), g[bad][:3], w[bad][:3])


def volume_of(kind, shape, seed):
    """(host volume for maps_host, input for the engine) of one dtype code."""
    import torch
    rng = np.random.default_rng(seed)
    ct = rng.integers(-1000, -600, shape)
    if kind in ("uint8", "int8"):
        v = rng.integers(0 if kind == "uint8" else -128, 256 if kind == "uint8" else 128, shape).astype(kind)
        return v, v
    if kind in ("int16", "int32", "int64"):
        v = ct.astype(kind)
        return v, v
    f = (ct + rng.random(shape)).astype(np.float32)
    f[rng.random(shape) < 0.05] = np.nan
    if kind == "bfloat16":
        t = torch.from_numpy(f).to(torch.bfloat16)
        return t.float().numpy(), t
    v = f.astype(kind)
    return v, v


KINDS = ["uint8", "int8", "int16", "int32", "int64", "float16", "bfloat16", "float32", "float64"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("masked", [True, False])
def test_every_dtype_radius_and_kernel_mode(inf, kind, r, masked):
    shape = (5, 8, 9)
    host, dev = volume_of(kind, shape, 3 * r + 2 * masked + KINDS.index(kind))
    mask = np.random.default_rng(r).integers(0, 3, shape).astype(np.uint8)
    bw = 2 if kind in ("uint8", "int8") else 25
    kw = dict(kernel_radius=r, masked_kernel=masked, bin_width=bw)
    assert_bits(inf.texture_maps(dev, mask, **kw), tm.maps_host(host, mask, **kw), kind)


@pytest.mark.parametrize("cls", tm.CLASSES)
@pytest.mark.parametrize("r", [1, 2, 3])
def test_each_class_alone(inf, cls, r):
    vol = synth.phantom(6, 14, 15, seed=20 + r)
    mask = two_lungs(6, 14, 15)
    mask[:, 5:9, 5:9] = 1
    kw = dict(classes=(cls,), kernel_radius=r, init_value=float("nan"))
    assert_bits(inf.texture_maps(vol, mask, **kw), tm.maps_host(vol, mask, **kw), (cls, r))


@pytest.mark.parametrize("shape", [(1, 5, 6), (4, 1, 7), (3, 6, 1), (1, 1, 1), (2, 1, 1), (6, 7, 8)])
def test_odd_even_and_unit_extents(inf, shape):
    host, dev = volume_of("int16", shape, 17)
    mask = np.ones(shape, np.uint8)
    for r in (1, 3):
        kw = dict(kernel_radius=r, init_value=float("nan"))
        assert_bits(inf.texture_maps(dev, mask, **kw), tm.maps_host(host, mask, **kw), (shape, r))


@pytest.mark.parametrize("row", [7, "lung"])
def test_forty_label_mask(inf, row):
    shape = (8, 20, 21)
    vol = synth.phantom(*shape, seed=9)
    mask = np.random.default_rng(4).integers(0, 41, shape).astype(np.uint8)
    for r, masked in ((1, True), (2, False)):
        kw = dict(label=row, kernel_radius=r, masked_kernel=masked, init_value=-1.0)
        assert_bits(inf.texture_maps(vol, mask, **kw), tm.maps_host(vol, mask, **kw), (row, r))


def test_speckle_mask(inf):
    """Hundreds of one-voxel zones; NGTDM is NaN at isolated centres."""
    vol = synth.phantom(6, 20, 20, seed=3)
    mask = np.zeros(vol.shape, np.uint8)
    mask[::2, ::2, ::2] = 1
    mask[2:4, 4:8, 4:8] = 1
    for r in (1, 2):
        res = inf.texture_maps(vol, mask, kernel_radius=r)
        assert_bits(res, tm.maps_host(vol, mask, kernel_radius=r), r)
    res = inf.texture_maps(vol, mask, kernel_radius=1)
    assert np.isnan(res["ngtdm_Contrast"][0, 0, 0]) and not np.isnan(res["ngtdm_Contrast"][2, 5, 5])


def test_all_zero_mask_holds_init_value(inf):
    vol = synth.phantom(4, 16, 16, seed=2)
    for init in (0.0, float("nan"), 3.5):
        res = inf.texture_maps(vol, np.zeros(vol.shape, np.uint8), init_value=init)
        assert res.voxels == 0 and len(res.maps) == 51
        assert_bits(res, tm.maps_host(vol, np.zeros(vol.shape, np.uint8), init_value=init))


def test_uniform_roi_and_255_levels(inf):
    """A uniform 7^3 ROI (one 343-voxel zone, runs of 7) at r = 3, and a level map spanning Ng = 255 (checkerboard)."""
    mask = np.zeros((9, 9, 9), np.uint8)
    mask[1:8, 1:8, 1:8] = 1
    uni = np.full(mask.shape, -900, np.int16)
    assert_bits(inf.texture_maps(uni, mask, kernel_radius=3), tm.maps_host(uni, mask, kernel_radius=3), "uniform")
    z, y, x = np.indices(mask.shape)
    chk = np.where((z + y + x) % 2 == 0, 0, 254 * 25).astype(np.int16)
    chk[4, 4, 4] = 127 * 25
    for r in (1, 3):
        res = inf.texture_maps(chk, mask, kernel_radius=r)
        assert res.n_levels == 255
        assert_bits(res, tm.maps_host(chk, mask, kernel_radius=r), ("checkerboard", r))


@pytest.mark.parametrize("alpha", [1, 3])
def test_gldm_alpha(inf, alpha):
    vol = synth.phantom(6, 18, 18, seed=40 + alpha)
    mask = two_lungs(6, 18, 18)
    kw = dict(classes=("gldm",), kernel_radius=2, bin_width=10, gldm_alpha=alpha)
    assert_bits(inf.texture_maps(vol, mask, **kw), tm.maps_host(vol, mask, **kw), alpha)


def test_feature_subset_is_the_full_planes(inf):
    vol = synth.phantom(8, 24, 24, seed=5)
    mask = two_lungs(8, 24, 24)
    full = inf.texture_maps(vol, mask, kernel_radius=2)
    names = ("ngtdm_Strength", "glszm_ZoneEntropy", "gldm_DependenceEntropy", "glrlm_RunVariance")
    sub = inf.texture_maps(vol, mask, kernel_radius=2, features=names)
    assert list(sub.maps) == ["glszm_ZoneEntropy", "glrlm_RunVariance", "gldm_DependenceEntropy", "ngtdm_Strength"]
    for k, m in sub.maps.items():
        assert np.array_equal(m.view(np.uint64), full[k].view(np.uint64))


def test_cover_case_equals_texture_row(inf):
    """A ROI inside an (r+1)^3 cube: every window holds the whole ROI, so every map equals the row's features."""
    rng = np.random.default_rng(8)
    vol = rng.integers(-1000, -800, (9, 10, 11)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    mask[3:6, 4:7, 4:7] = rng.integers(0, 2, (3, 3, 3)).astype(np.uint8) * 2
    mask[4, 5, 5] = 2
    res = inf.texture_maps(vol, mask, label=2, kernel_radius=2)
    row = next(t for t in inf.texture(vol, mask, classes=tm.CLASSES).rows if t.label == 2)
    for cls in tm.CLASSES:
        for k, want in getattr(row, cls).items():
            got = res["%s_%s" % (cls, k)][mask == 2]
            assert np.allclose(got, want, rtol=1e-12, atol=1e-12), (cls, k)


def test_cuda_cpu_tensor_and_numpy_agree(inf):
    import torch
    vol = synth.phantom(6, 32, 34, seed=12)
    mask = two_lungs(6, 32, 34)
    a = inf.texture_maps(_cuda(vol), _cuda(mask), label=1, kernel_radius=2)
    b = inf.texture_maps(torch.from_numpy(vol), torch.from_numpy(mask), label=1, kernel_radius=2)
    c = inf.texture_maps(vol, mask, label=1, kernel_radius=2)
    for k in c.maps:
        assert a[k].is_cuda and a[k].dtype == torch.float64 and tuple(a[k].shape) == vol.shape
        assert isinstance(b[k], torch.Tensor) and not b[k].is_cuda
        assert isinstance(c[k], np.ndarray)
        assert np.array_equal(a[k].cpu().numpy().view(np.uint64), c[k].view(np.uint64))
        assert np.array_equal(b[k].numpy().view(np.uint64), c[k].view(np.uint64))


def test_wavelet_band_as_input(inf):
    vol = synth.phantom(8, 20, 22, seed=31)
    mask = two_lungs(8, 20, 22)
    band = inf.wavelet(vol, decompositions=("wavelet-LLL",))["wavelet-LLL"]
    kw = dict(kernel_radius=1, bin_width=50, masked_kernel=False)
    assert_bits(inf.texture_maps(band, mask, **kw), tm.maps_host(band, mask, **kw))


def test_refusals(inf, monkeypatch):
    from lungmask_b200 import _native
    vol = synth.phantom(6, 20, 20, seed=14).astype(np.float32)
    mask = two_lungs(6, 20, 20)

    def no_kernel(*a, **k):
        raise AssertionError("a map kernel ran")
    monkeypatch.setattr(inf.engine, "texture_maps_dev", no_kernel)
    bad = vol.copy()
    bad[mask == 1] = np.where(np.arange((mask == 1).sum()) == 3, np.inf, bad[mask == 1])
    with pytest.raises(ValueError, match="non-finite"):
        inf.texture_maps(bad, mask)
    with pytest.raises(ValueError, match="grey levels"):
        inf.texture_maps(vol * 100, mask, bin_width=1)
    with pytest.raises(ValueError, match="kernel_radius"):
        inf.texture_maps(vol, mask, kernel_radius=4)
    with pytest.raises(ValueError, match="unknown feature"):
        inf.texture_maps(vol, mask, features=("glszm_ZoneEntropy", "glszm_Bogus"))
    with pytest.raises(ValueError, match="glcm_maps"):
        inf.texture_maps(vol, mask, classes=("glcm",))
    with pytest.raises(ValueError, match="gldm_alpha"):
        inf.texture_maps(vol, mask, gldm_alpha=-1)
    with pytest.raises(ValueError, match="label"):
        inf.texture_maps(vol, mask, label=0)
    monkeypatch.undo()
    levels = np.zeros(vol.shape, np.uint8)
    levels[mask > 0] = 3
    tl, tmk = _cuda(levels), _cuda(mask)
    table = _cuda(fm.entropy_table(27))
    out = _cuda(np.zeros((1,) + vol.shape))
    e = inf.engine

    def call(lv=tl, **over):
        a = dict(row=256, radius=1, n_levels=5, cls=1, alpha=0, init_value=0.0, feature_bits=1 << 11,
                 d_table_ptr=table.data_ptr(), table_len=378, d_out_ptr=out.data_ptr())
        a.update(over)
        e.texture_maps_dev(lv.data_ptr(), tmk.data_ptr(), vol.shape, **a)
    call()
    assert (out[0][_cuda(mask) > 0] == 3 * 3).all()   # HighGrayLevelZoneEmphasis of a single level 3
    for over, msg in ((dict(radius=4), "radius"), (dict(row=0), "row"), (dict(cls=0), "class"), (dict(cls=5), "class"),
                      (dict(alpha=-1), "alpha"), (dict(feature_bits=0), "feature_bits"),
                      (dict(feature_bits=1 << 16), "feature_bits"), (dict(cls=3, feature_bits=1 << 14), "feature_bits"),
                      (dict(cls=4, feature_bits=1 << 5), "feature_bits"), (dict(table_len=377), "table_len"),
                      (dict(n_levels=256), "n_levels"), (dict(n_levels=0), "n_levels"),
                      (dict(d_out_ptr=tl.data_ptr()), "overlaps"), (dict(d_out_ptr=table.data_ptr()), "overlaps")):
        with pytest.raises(_native.NativeError, match=msg):
            call(**over)
    high = levels.copy()
    high[3, 10, 10] = 9   # a level above n_levels = 5
    for cls in (1, 2, 3, 4):
        with pytest.raises(_native.NativeError, match="above n_levels"):
            call(lv=_cuda(high), cls=cls, feature_bits=1)


@pytest.mark.parametrize("r", [1, 2])
def test_full_size_phantom(inf, r):
    """The 300 x 512 x 512 two-lung phantom: the first and last 4 slices, a slice near the apex and, at r = 1, one middle
    slice (the numpy statement's cost, about 20 s per 10^5 ROI voxels at r = 1 for the four classes, bounds the middle)."""
    vol = synth.phantom(300, 512, 512, seed=100)
    mask = two_lungs(300, 512, 512)
    res = inf.texture_maps(_cuda(vol), _cuda(mask), kernel_radius=r)
    assert res.voxels == int((mask > 0).sum())
    ranges = ((0, 4), (20, 21), (296, 300)) + (((150, 151),) if r == 1 else ())
    for lo, hi in ranges:
        want = tm.maps_host(vol, mask, kernel_radius=r, slices=range(lo, hi))
        assert (want.low, want.n_levels) == (res.low, res.n_levels)
        for k, m in res.maps.items():
            g = m[lo:hi].cpu().numpy()
            assert np.array_equal(g.view(np.uint64), want[k][lo:hi].view(np.uint64)), (lo, k)


def test_cli_writes_maps(tmp_path):
    import torch
    from lungmask_b200.__main__ import main
    from lungmask_b200.io import load_input_image
    p = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.npy")
    vol = synth.phantom(6, 96, 96, seed=21)
    np.save(src, vol)
    out = tmp_path / "maps"
    names = ("glszm_ZoneEntropy", "ngtdm_Coarseness")
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--texture-maps", str(out),
          "--texture-maps-classes", "ngtdm,glszm", "--texture-maps-features", ",".join(names),
          "--texture-maps-radius", "2", "--texture-bin-width", "50"])
    mask = np.load(str(tmp_path / "m.npy"))
    want = tm.maps_host(vol, mask, classes=("glszm", "ngtdm"), features=names, kernel_radius=2, bin_width=50)
    assert sorted(f.name for f in out.iterdir()) == ["lung_glszm_ZoneEntropy.nii.gz", "lung_ngtdm_Coarseness.nii.gz"]
    for k in names:
        img = load_input_image(str(out / ("lung_%s.nii.gz" % k)))
        assert np.array_equal(np.asarray(img.array).view(np.uint64), want[k].view(np.uint64))
    assert tx.NGTDM_FEATURES[0] == "Coarseness"
