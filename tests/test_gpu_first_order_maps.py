"""Voxel-based first-order maps on the GPU (LMInferer.first_order_maps, lm_first_order_maps_dev): every map bit for bit
(uint64 patterns) against the numpy statement first_order_maps.maps_host."""
import numpy as np
import pytest

from lungmask_b200 import first_order as fo
from lungmask_b200 import first_order_maps as fm
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


def two_lungs(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


def assert_bits(got, want, where=""):
    """Every plane of two FirstOrderMaps equal as uint64 patterns."""
    assert list(got.maps) == list(want.maps)
    assert (got.low, got.n_levels, got.exact, got.voxels) == (want.low, want.n_levels, want.exact, want.voxels), where
    for k, m in got.maps.items():
        g = np.ascontiguousarray(m.cpu().numpy() if hasattr(m, "cpu") else m)
        w = want.maps[k]
        bad = g.view(np.uint64) != w.view(np.uint64)
        assert not bad.any(), (where, k, int(bad.sum()), g[bad][:3], w[bad][:3])


def volume_of(kind, shape, seed):
    """(host volume for maps_host, input for the engine) of one dtype code."""
    import torch
    rng = np.random.default_rng(seed)
    ct = rng.integers(-1000, 300, shape)
    if kind in ("uint8", "int8"):
        v = rng.integers(0 if kind == "uint8" else -128, 256 if kind == "uint8" else 128, shape).astype(kind)
        return v, v
    if kind in ("int16", "int32", "int64"):
        v = ct.astype(kind)
        return v, v
    if kind == "int32wide":
        v = rng.integers(-(1 << 23), 1 << 23, shape).astype(np.int32)
        return v, v
    f = (ct + rng.random(shape)).astype(np.float32)
    f[rng.random(shape) < 0.05] = np.nan
    f.reshape(-1)[:3] = (-0.0, 0.0, -0.0)[:f.size]
    if kind == "bfloat16":
        t = torch.from_numpy(f).to(torch.bfloat16)
        return t.float().numpy(), t
    v = f.astype(kind)
    return v, v


KINDS = ["uint8", "int8", "int16", "int32", "int32wide", "int64", "float16", "bfloat16", "float32", "float64"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("masked", [True, False])
def test_every_dtype_radius_and_kernel_mode(inf, kind, r, masked):
    shape = (6, 9, 10)
    host, dev = volume_of(kind, shape, 3 * r + 2 * masked + KINDS.index(kind))
    mask = np.random.default_rng(r).integers(0, 3, shape).astype(np.uint8)
    bw = (1 << 17) if kind == "int32wide" else (2 if kind in ("uint8", "int8") else 25)
    kw = dict(kernel_radius=r, masked_kernel=masked, bin_width=bw, voxel_array_shift=-5, spacing=(0.7, 0.8, 2.5))
    want = fm.maps_host(host, mask, **kw)
    assert want.exact == (kind in ("uint8", "int8", "int16", "int32", "int64"))
    assert_bits(inf.first_order_maps(dev, mask, **kw), want, kind)


@pytest.mark.parametrize("shape", [(1, 5, 6), (4, 1, 7), (3, 6, 1), (1, 1, 1), (2, 1, 1), (7, 8, 9)])
@pytest.mark.parametrize("kind", ["int16", "float32"])
def test_odd_even_and_unit_extents(inf, shape, kind):
    host, dev = volume_of(kind, shape, 17)
    mask = np.ones(shape, np.uint8)
    for r in (1, 3):
        kw = dict(kernel_radius=r, init_value=float("nan"))
        assert_bits(inf.first_order_maps(dev, mask, **kw), fm.maps_host(host, mask, **kw), (shape, r))


@pytest.mark.parametrize("row", [7, "lung"])
def test_forty_label_mask(inf, row):
    shape = (12, 30, 31)
    vol = synth.phantom(*shape, seed=9)
    mask = np.random.default_rng(4).integers(0, 41, shape).astype(np.uint8)
    for r, masked in ((1, True), (2, False)):
        kw = dict(label=row, kernel_radius=r, masked_kernel=masked, init_value=-1.0)
        assert_bits(inf.first_order_maps(vol, mask, **kw), fm.maps_host(vol, mask, **kw), (row, r))


def test_all_zero_mask_holds_init_value(inf):
    vol = synth.phantom(4, 16, 16, seed=2)
    for init in (0.0, float("nan"), 3.5):
        res = inf.first_order_maps(vol, np.zeros(vol.shape, np.uint8), init_value=init)
        assert res.voxels == 0 and len(res.maps) == 18
        assert_bits(res, fm.maps_host(vol, np.zeros(vol.shape, np.uint8), init_value=init))


def test_feature_subset_is_the_full_planes(inf):
    vol = synth.phantom(8, 32, 32, seed=5)
    mask = two_lungs(8, 32, 32)
    full = inf.first_order_maps(vol, mask, kernel_radius=2)
    sub = inf.first_order_maps(vol, mask, kernel_radius=2, features=("Variance", "Entropy", "Mean"))
    assert list(sub.maps) == ["Entropy", "Mean", "Variance"]
    for k, m in sub.maps.items():
        assert np.array_equal(m.view(np.uint64), full[k].view(np.uint64))


def test_cuda_cpu_tensor_and_numpy_agree(inf):
    import torch
    vol = synth.phantom(8, 40, 44, seed=12)
    mask = two_lungs(8, 40, 44)
    a = inf.first_order_maps(_cuda(vol), _cuda(mask), label=1, kernel_radius=2)
    b = inf.first_order_maps(torch.from_numpy(vol), torch.from_numpy(mask), label=1, kernel_radius=2)
    c = inf.first_order_maps(vol, mask, label=1, kernel_radius=2)
    for k in fo.FIRST_ORDER_FEATURES:
        assert a[k].is_cuda and a[k].dtype == torch.float64 and tuple(a[k].shape) == vol.shape
        assert isinstance(b[k], torch.Tensor) and not b[k].is_cuda
        assert isinstance(c[k], np.ndarray)
        assert np.array_equal(a[k].cpu().numpy().view(np.uint64), c[k].view(np.uint64))
        assert np.array_equal(b[k].numpy().view(np.uint64), c[k].view(np.uint64))


def test_wavelet_band_as_input(inf):
    vol = synth.phantom(8, 24, 26, seed=31)
    mask = two_lungs(8, 24, 26)
    band = inf.wavelet(vol, decompositions=("wavelet-LLL",))["wavelet-LLL"]
    kw = dict(kernel_radius=1, bin_width=50)
    res = inf.first_order_maps(band, mask, **kw)
    assert not res.exact
    assert_bits(res, fm.maps_host(band, mask, **kw))


def test_refusals(inf, monkeypatch):
    from lungmask_b200 import _native
    vol = synth.phantom(6, 20, 20, seed=14).astype(np.float32)
    mask = two_lungs(6, 20, 20)

    def no_kernel(*a, **k):
        raise AssertionError("a map kernel ran")
    monkeypatch.setattr(inf.engine, "first_order_maps_dev", no_kernel)
    bad = vol.copy()
    bad[mask == 1] = np.where(np.arange((mask == 1).sum()) == 3, np.inf, bad[mask == 1])
    with pytest.raises(ValueError, match="non-finite"):
        inf.first_order_maps(bad, mask)
    with pytest.raises(ValueError, match="grey levels"):
        inf.first_order_maps(vol * 100, mask, bin_width=1)
    with pytest.raises(ValueError, match="kernel_radius"):
        inf.first_order_maps(vol, mask, kernel_radius=4)
    with pytest.raises(ValueError, match="unknown first-order feature"):
        inf.first_order_maps(vol, mask, features=("Mean", "Mode"))
    with pytest.raises(ValueError, match="label"):
        inf.first_order_maps(vol, mask, label=0)
    with pytest.raises(ValueError, match="2\\^58"):
        inf.first_order_maps(vol.astype(np.int16), mask, voxel_array_shift=1 << 58)
    monkeypatch.undo()
    tv, tm = _cuda(vol), _cuda(mask)
    table = _cuda(fm.entropy_table(27))
    out = _cuda(np.zeros((1,) + vol.shape))
    e = inf.engine

    def call(**over):
        a = dict(row=256, radius=1, masked=True, bin_width=25, low=-1000, n_levels=40, exact=False, base=0, shift=0,
                 voxel_volume=float("nan"), init_value=0.0, feature_bits=1, d_table_ptr=table.data_ptr(), table_len=378,
                 d_out_ptr=out.data_ptr())
        a.update(over)
        e.first_order_maps_dev(tv.data_ptr(), _native.DTYPE_F32, tm.data_ptr(), vol.shape, **a)
    call()
    for over, msg in ((dict(radius=4), "radius"), (dict(row=0), "row"), (dict(feature_bits=0), "feature_bits"),
                      (dict(feature_bits=1 << 18), "feature_bits"), (dict(table_len=377), "table_len"),
                      (dict(exact=True), "integer volume"), (dict(n_levels=256), "n_levels"),
                      (dict(bin_width=0), "bin_width"), (dict(voxel_volume=-1.0), "voxel_volume"),
                      (dict(d_out_ptr=tv.data_ptr()), "overlaps"), (dict(shift=1 << 58), "shift")):
        with pytest.raises(_native.NativeError, match=msg):
            call(**over)


@pytest.mark.parametrize("r", [1, 2])
def test_full_size_phantom(inf, r):
    vol = synth.phantom(300, 512, 512, seed=100)
    mask = two_lungs(300, 512, 512)
    res = inf.first_order_maps(_cuda(vol), _cuda(mask), kernel_radius=r, spacing=(0.7, 0.7, 1.0))
    assert res.exact and res.voxels == int((mask > 0).sum())
    for lo in (0, 146, 292):
        want = fm.maps_host(vol, mask, kernel_radius=r, spacing=(0.7, 0.7, 1.0), slices=range(lo, lo + 8))
        for k, m in res.maps.items():
            g = m[lo:lo + 8].cpu().numpy()
            assert np.array_equal(g.view(np.uint64), want[k][lo:lo + 8].view(np.uint64)), (lo, k)


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
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--first-order-maps", str(out),
          "--first-order-maps-features", "Mean,Entropy", "--first-order-maps-radius", "2", "--first-order-shift", "10"])
    mask = np.load(str(tmp_path / "m.npy"))
    want = fm.maps_host(vol, mask, features=("Mean", "Entropy"), kernel_radius=2, voxel_array_shift=10)
    assert sorted(f.name for f in out.iterdir()) == ["lung_Entropy.nii.gz", "lung_Mean.nii.gz"]
    for k in ("Mean", "Entropy"):
        img = load_input_image(str(out / ("lung_%s.nii.gz" % k)))
        assert np.array_equal(np.asarray(img.array).view(np.uint64), want[k].view(np.uint64))
