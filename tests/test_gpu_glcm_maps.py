"""Voxel-based GLCM maps on the GPU (LMInferer.glcm_maps, lm_glcm_maps_dev): every map bit for bit (uint64 patterns)
against the numpy statement glcm_maps.maps_host."""
import numpy as np
import pytest

from lungmask_b200 import first_order_maps as fm
from lungmask_b200 import glcm_maps as gm
from lungmask_b200 import texture as tx
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
    """Every plane of two GLCMMaps equal as uint64 patterns."""
    assert list(got.maps) == list(want.maps)
    assert (got.low, got.n_levels, got.voxels) == (want.low, want.n_levels, want.voxels), where
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
    assert_bits(inf.glcm_maps(dev, mask, **kw), gm.maps_host(host, mask, **kw), kind)


@pytest.mark.parametrize("shape", [(1, 5, 6), (4, 1, 7), (3, 6, 1), (1, 1, 1), (2, 1, 1), (6, 7, 8)])
def test_odd_even_and_unit_extents(inf, shape):
    host, dev = volume_of("int16", shape, 17)
    mask = np.ones(shape, np.uint8)
    for r in (1, 3):
        kw = dict(kernel_radius=r, init_value=float("nan"))
        assert_bits(inf.glcm_maps(dev, mask, **kw), gm.maps_host(host, mask, **kw), (shape, r))


@pytest.mark.parametrize("row", [7, "lung"])
def test_forty_label_mask(inf, row):
    shape = (10, 24, 25)
    vol = synth.phantom(*shape, seed=9)
    mask = np.random.default_rng(4).integers(0, 41, shape).astype(np.uint8)
    for r, masked in ((1, True), (2, False)):
        kw = dict(label=row, kernel_radius=r, masked_kernel=masked, init_value=-1.0)
        assert_bits(inf.glcm_maps(vol, mask, **kw), gm.maps_host(vol, mask, **kw), (row, r))


def test_speckle_mask_gives_nan_at_isolated_voxels(inf):
    vol = synth.phantom(6, 20, 20, seed=3)
    mask = np.zeros(vol.shape, np.uint8)
    mask[::2, ::2, ::2] = 1
    mask[2:4, 4:8, 4:8] = 1
    res = inf.glcm_maps(vol, mask, kernel_radius=1)
    assert_bits(res, gm.maps_host(vol, mask, kernel_radius=1))
    assert np.isnan(res["Contrast"][0, 0, 0]) and not np.isnan(res["Contrast"][2, 5, 5])


def test_all_zero_mask_holds_init_value(inf):
    vol = synth.phantom(4, 16, 16, seed=2)
    for init in (0.0, float("nan"), 3.5):
        res = inf.glcm_maps(vol, np.zeros(vol.shape, np.uint8), init_value=init)
        assert res.voxels == 0 and len(res.maps) == 22
        assert_bits(res, gm.maps_host(vol, np.zeros(vol.shape, np.uint8), init_value=init))


def test_feature_subset_is_the_full_planes(inf):
    vol = synth.phantom(8, 32, 32, seed=5)
    mask = two_lungs(8, 32, 32)
    full = inf.glcm_maps(vol, mask, kernel_radius=2)
    sub = inf.glcm_maps(vol, mask, kernel_radius=2, features=("Imc2", "Contrast", "JointEntropy"))
    assert list(sub.maps) == ["Contrast", "JointEntropy", "Imc2"]
    for k, m in sub.maps.items():
        assert np.array_equal(m.view(np.uint64), full[k].view(np.uint64))


def test_cover_case_equals_texture_row(inf):
    """A ROI inside an (r+1)^3 cube: every window holds the whole ROI, so every map equals the row's GLCM features."""
    rng = np.random.default_rng(8)
    vol = rng.integers(-1000, -500, (9, 10, 11)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    mask[3:6, 4:7, 4:7] = rng.integers(0, 2, (3, 3, 3)).astype(np.uint8) * 2
    mask[4, 5, 5] = 2
    res = inf.glcm_maps(vol, mask, label=2, kernel_radius=2)
    row = next(t for t in inf.texture(vol, mask, classes=("glcm",)).rows if t.label == 2)
    for k in gm.FEATURES:
        got = res[k][mask == 2]
        assert np.allclose(got, row.glcm[k], rtol=1e-12, atol=1e-12), k


def test_cuda_cpu_tensor_and_numpy_agree(inf):
    import torch
    vol = synth.phantom(8, 40, 44, seed=12)
    mask = two_lungs(8, 40, 44)
    a = inf.glcm_maps(_cuda(vol), _cuda(mask), label=1, kernel_radius=2)
    b = inf.glcm_maps(torch.from_numpy(vol), torch.from_numpy(mask), label=1, kernel_radius=2)
    c = inf.glcm_maps(vol, mask, label=1, kernel_radius=2)
    for k in gm.FEATURES:
        assert a[k].is_cuda and a[k].dtype == torch.float64 and tuple(a[k].shape) == vol.shape
        assert isinstance(b[k], torch.Tensor) and not b[k].is_cuda
        assert isinstance(c[k], np.ndarray)
        assert np.array_equal(a[k].cpu().numpy().view(np.uint64), c[k].view(np.uint64))
        assert np.array_equal(b[k].numpy().view(np.uint64), c[k].view(np.uint64))


def test_wavelet_band_as_input(inf):
    vol = synth.phantom(8, 24, 26, seed=31)
    mask = two_lungs(8, 24, 26)
    band = inf.wavelet(vol, decompositions=("wavelet-LLL",))["wavelet-LLL"]
    kw = dict(kernel_radius=1, bin_width=50, masked_kernel=False)
    assert_bits(inf.glcm_maps(band, mask, **kw), gm.maps_host(band, mask, **kw))


def test_refusals(inf, monkeypatch):
    from lungmask_b200 import _native
    vol = synth.phantom(6, 20, 20, seed=14).astype(np.float32)
    mask = two_lungs(6, 20, 20)

    def no_kernel(*a, **k):
        raise AssertionError("a map kernel ran")
    monkeypatch.setattr(inf.engine, "glcm_maps_dev", no_kernel)
    bad = vol.copy()
    bad[mask == 1] = np.where(np.arange((mask == 1).sum()) == 3, np.inf, bad[mask == 1])
    with pytest.raises(ValueError, match="non-finite"):
        inf.glcm_maps(bad, mask)
    with pytest.raises(ValueError, match="grey levels"):
        inf.glcm_maps(vol * 100, mask, bin_width=1)
    with pytest.raises(ValueError, match="kernel_radius"):
        inf.glcm_maps(vol, mask, kernel_radius=4)
    with pytest.raises(ValueError, match="unknown GLCM feature"):
        inf.glcm_maps(vol, mask, features=("Contrast", "MCC"))
    with pytest.raises(ValueError, match="label"):
        inf.glcm_maps(vol, mask, label=0)
    monkeypatch.undo()
    levels = np.zeros(vol.shape, np.uint8)
    levels[mask > 0] = 3
    tl, tm = _cuda(levels), _cuda(mask)
    table = _cuda(fm.entropy_table(36))
    out = _cuda(np.zeros((1,) + vol.shape))
    e = inf.engine

    def call(lv=tl, **over):
        a = dict(row=256, radius=1, n_levels=5, init_value=0.0, feature_bits=1, d_table_ptr=table.data_ptr(),
                 table_len=666, d_out_ptr=out.data_ptr())
        a.update(over)
        e.glcm_maps_dev(lv.data_ptr(), tm.data_ptr(), vol.shape, **a)
    call()
    assert (out[0][_cuda(mask) > 0] == 3 * 3).all()   # Autocorrelation of a single level 3
    for over, msg in ((dict(radius=4), "radius"), (dict(row=0), "row"), (dict(feature_bits=0), "feature_bits"),
                      (dict(feature_bits=1 << 22), "feature_bits"), (dict(table_len=665), "table_len"),
                      (dict(n_levels=256), "n_levels"), (dict(n_levels=0), "n_levels"),
                      (dict(d_out_ptr=tl.data_ptr()), "overlaps"), (dict(d_out_ptr=table.data_ptr()), "overlaps")):
        with pytest.raises(_native.NativeError, match=msg):
            call(**over)
    high = levels.copy()
    high[3, 10, 10] = 9   # a level above n_levels = 5
    with pytest.raises(_native.NativeError, match="above n_levels"):
        call(lv=_cuda(high))


@pytest.mark.parametrize("r", [1, 2])
def test_full_size_phantom(inf, r):
    """The 300 x 512 x 512 two-lung phantom: the first and last 8 slices, and 2 middle slices (the numpy statement's
    cost bounds the middle)."""
    vol = synth.phantom(300, 512, 512, seed=100)
    mask = two_lungs(300, 512, 512)
    res = inf.glcm_maps(_cuda(vol), _cuda(mask), kernel_radius=r)
    assert res.voxels == int((mask > 0).sum())
    for lo, hi in ((0, 8), (149, 151), (292, 300)):
        want = gm.maps_host(vol, mask, kernel_radius=r, slices=range(lo, hi))
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
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--glcm-maps", str(out),
          "--glcm-maps-features", "Contrast,Idm", "--glcm-maps-radius", "2", "--texture-bin-width", "50"])
    mask = np.load(str(tmp_path / "m.npy"))
    want = gm.maps_host(vol, mask, features=("Contrast", "Idm"), kernel_radius=2, bin_width=50)
    assert sorted(f.name for f in out.iterdir()) == ["lung_glcm_Contrast.nii.gz", "lung_glcm_Idm.nii.gz"]
    for k in ("Contrast", "Idm"):
        img = load_input_image(str(out / ("lung_glcm_%s.nii.gz" % k)))
        assert np.array_equal(np.asarray(img.array).view(np.uint64), want[k].view(np.uint64))
    assert tx.GLCM_FEATURES.index("Contrast") < tx.GLCM_FEATURES.index("Idm")
