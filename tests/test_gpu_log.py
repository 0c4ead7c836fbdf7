"""The LoG image type on the GPU (LMInferer.log_images, LMInferer.log_features; lm_laplacian_of_gaussian_dev) against
the numpy statement lungmask_b200.laplacian.log_host: the image as uint64 bit patterns for every dtype code, odd
extents, extents of exactly 4 and exactly ceil(sigma / s) + 1, sigma / s below 1 and above 4, anisotropic spacing and
the 300x512x512 phantom; the features against first_order and texture on the host-stated image; every input kind; the
refusals; and --log on the command line against the same chain in Python."""
import json
import math
import os

import numpy as np
import pytest

from lungmask_b200 import laplacian as lg
from oracle import synth

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 1.25)   # (x, y, z) mm


@pytest.fixture(scope="module")
def inf():
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=71, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def bits(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    assert a.dtype == np.float64
    return np.ascontiguousarray(a).view(np.uint64)


def two_lungs(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


def five_lobes(mask):
    S, H, _ = mask.shape
    z, y, _ = np.ogrid[:S, :H, :1]
    lobes = mask.copy()
    lobes[(mask == 1) & (z >= S // 2)] = 2
    lobes[(mask == 1) & (z >= S // 2) & (y >= H // 2)] = 3
    lobes[(mask == 2) & (z < S // 2)] = 4
    lobes[(mask == 2) & (z >= S // 2)] = 5
    return lobes


def check_images(got, ref, sigmas, spacing, what):
    assert list(got) == [lg.image_name(s) for s in sigmas], what
    for s in sigmas:
        want = lg.log_host(ref, s, spacing)
        assert np.array_equal(bits(got[lg.image_name(s)]), bits(want)), (what, s)


# ---- images

def _values(dtype, shape, seed):
    import torch
    rng = np.random.default_rng(seed)
    if dtype == torch.bool:
        return torch.from_numpy(rng.random(shape) < 0.4)
    if dtype in (torch.uint8, torch.int8):
        info = np.iinfo(np.uint8 if dtype == torch.uint8 else np.int8)
        return torch.from_numpy(rng.integers(info.min, info.max + 1, shape).astype(np.int64)).to(dtype)
    if dtype in (torch.int16, torch.int32, torch.int64):
        hi = {torch.int16: 32767, torch.int32: 2 ** 31 - 1, torch.int64: 2 ** 53}[dtype]
        return torch.from_numpy(rng.integers(-hi, hi, shape, dtype=np.int64)).to(dtype)
    x = torch.from_numpy(rng.standard_normal(shape) * 900.0)
    x[0, 0, :2] = torch.tensor([0.0, -0.0], dtype=torch.float64)
    return x.to(dtype)


def test_images_every_dtype_code(inf):
    import torch
    shape = (7, 10, 37)
    for k, dtype in enumerate((torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16,
                               torch.bfloat16, torch.float32, torch.float64, torch.bool)):
        t = _values(dtype, shape, 300 + k)
        ref = t.double().numpy()
        check_images(inf.log_images(t.cuda(), (1.0, 2.5), spacing=SPACING), ref, (1.0, 2.5), SPACING, (dtype, "cuda"))
        check_images(inf.log_images(t, 1.5, spacing=SPACING), ref, (1.5,), SPACING, (dtype, "cpu tensor"))


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_images_extents_and_scales(inf, dtype):
    """Odd extents, extents of exactly 4 and of exactly ceil(sigma / s) + 1, sigma / s from 0.3 to 7, anisotropic."""
    cases = [((4, 4, 4), (1.0, 1.0, 1.0), (0.3, 1.0, 3.0), 3.01),          # 4 = ceil(3 / 1) + 1
             ((5, 9, 33), (0.7, 0.8, 2.5), (0.75, 2.0, 5.0), 6.5),          # 8 = ceil(5 / 0.8) + 1 <= 9
             ((17, 31, 65), (0.7, 0.7, 1.25), (0.5, 4.0, 5.0), 40.0),       # sigma / s from 0.4 to 7.1
             ((6, 9, 9), (1.0, 1.0, 1.0), (5.0,), 5.05),                    # 6 = ceil(5) + 1
             ((9, 9, 9), (1.0, 1.0, 1.0), (8.0, 7.5), 8.08),                # 9 = ceil(8) + 1 = ceil(7.5) + 1
             ((5, 13, 16), (1.0, 0.5, 1.5), (6.0,), 6.06),                  # 5 = ceil(6 / 1.5) + 1, 13 = ceil(12) + 1
             ((130, 6, 5), (2.0, 1.0, 0.25), (5.0, 2.5), 5.5)]              # 6 = ceil(5 / 1) + 1, z lines of 130
    for i, (shape, spacing, sigmas, too_big) in enumerate(cases):
        rng = np.random.default_rng(i)
        vol = rng.integers(-1024, 2000, shape).astype(dtype)
        if dtype == np.float32:
            vol = vol + rng.random(shape).astype(np.float32)
        check_images(inf.log_images(vol, sigmas, spacing=spacing), vol, sigmas, spacing, (dtype, shape))
        with pytest.raises(ValueError, match="ceil"):
            inf.log_images(vol, sigmas + (too_big,), spacing=spacing)


def test_images_of_the_300x512x512_phantom(inf):
    """The whole image at sigma 1 and 5 mm of the int16 phantom, bit for bit; one image on the host at a time."""
    vol = synth.phantom(300, 512, 512, seed=31)
    tv = _cuda(vol)
    for s in (1.0, 5.0):
        got = inf.log_images(tv, s, spacing=SPACING)[lg.image_name(s)]
        want = lg.log_host(vol, s, SPACING)
        assert np.array_equal(bits(got), bits(want)), s
        del got, want
    assert np.array_equal(tv.cpu().numpy(), vol)


# ---- input kinds and streams

def test_input_kinds_agree(inf):
    import torch
    from lungmask_b200.io import Volume
    vol = np.random.default_rng(3).integers(-1024, 600, (12, 20, 22)).astype(np.int16)
    keep = vol.copy()
    sp = (1.0, 1.0, 2.0)
    sig = (1.0, 3.0)
    from_np = inf.log_images(vol, sig, spacing=sp)
    from_cpu = inf.log_images(torch.from_numpy(vol), sig, spacing=sp)
    t = _cuda(vol)
    from_cuda = inf.log_images(t, sig, spacing=sp)
    from_volume = inf.log_images(Volume(vol, spacing=sp), sig)   # the Volume supplies the spacing
    assert np.array_equal(vol, keep) and np.array_equal(t.cpu().numpy(), keep)
    for s in sig:
        name = lg.image_name(s)
        a = from_np[name]
        assert isinstance(a, np.ndarray) and a.dtype == np.float64
        b, c = from_cpu[name], from_cuda[name]
        assert isinstance(b, torch.Tensor) and b.device.type == "cpu" and b.dtype == torch.float64
        assert c.is_cuda and c.device.index == inf.engine.device and c.dtype == torch.float64
        assert isinstance(from_volume[name], np.ndarray)
        for other in (b, c, from_volume[name]):
            assert np.array_equal(bits(a), bits(other)), name
        assert np.array_equal(bits(a), bits(lg.log_host(vol, s, sp)))
    assert len({from_cuda[lg.image_name(s)].data_ptr() for s in sig}) == 2


def test_cuda_inputs_read_after_work_on_the_callers_stream(inf):
    import torch
    vol = synth.phantom(16, 64, 64, seed=12)
    mask = two_lungs(*vol.shape)
    src, msrc = _cuda(vol), _cuda(mask)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.zeros_like(src)
        m = torch.zeros_like(msrc)
        torch.cuda._sleep(20_000_000)   # the copies below are still queued when the calls are made
        t.copy_(src)
        m.copy_(msrc)
        got = inf.log_images(t, (1.0, 2.0), spacing=SPACING)
        feats = inf.log_features(t, m, (1.0, 2.0), classes=("glcm",), spacing=SPACING)
    side.synchronize()
    check_images(got, vol, (1.0, 2.0), SPACING, "stream")
    want = inf.log_features(vol, mask, (1.0, 2.0), classes=("glcm",), spacing=SPACING)
    for d, e in zip(feats.images, want.images):
        assert json.dumps(d.texture.to_dict()) == json.dumps(e.texture.to_dict()), d.name


# ---- refusals, before any kernel

def test_refusals_before_any_kernel(inf, monkeypatch):
    calls = []
    orig = inf.engine.laplacian_of_gaussian_dev
    monkeypatch.setattr(inf.engine, "laplacian_of_gaussian_dev",
                        lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
    vol = np.random.default_rng(4).standard_normal((8, 9, 10)).astype(np.float32)
    mask = (np.abs(vol) < 1).astype(np.uint8)
    for x in (vol, _cuda(vol)):
        for bad in ([], [0.0], [-1.0], [math.nan], [math.inf], [1.0, 1]):
            with pytest.raises(ValueError, match="sigma"):
                inf.log_images(x, bad, spacing=SPACING)
        with pytest.raises(ValueError, match="spacing is needed"):
            inf.log_images(x, 1.0)
        with pytest.raises(ValueError, match="spacing"):
            inf.log_images(x, 1.0, spacing=(1.0, 0.0, 1.0))
        inf.log_images(x, 7.0, spacing=(1.0, 1.0, 1.0)) if x is vol else None   # 8 slices = ceil(7) + 1
        with pytest.raises(ValueError, match="along z"):
            inf.log_images(x, 7.5, spacing=(1.0, 1.0, 1.0))     # 8 slices < ceil(7.5) + 1
        with pytest.raises(ValueError, match="under 4"):
            inf.log_images(x[:3], 1.0, spacing=SPACING)
    with pytest.raises(ValueError, match="spacing is needed"):
        inf.log_features(vol, mask, 1.0)
    with pytest.raises(ValueError, match="no bin width"):
        inf.log_features(vol, mask, (1.0, 2.0), bin_width={1.0: 25}, spacing=SPACING)
    with pytest.raises(ValueError, match="unknown feature class"):
        inf.log_features(vol, mask, 1.0, classes=("glcm", "shape"), spacing=SPACING)
    assert calls == [1]   # the one call that fits
    with pytest.raises(ValueError, match="log"):   # the ABI's own checks
        inf.engine.laplacian_of_gaussian_dev(_cuda(vol).data_ptr(), 1, (8, 9, 3), SPACING, 1.0, (0, 0), 0)
    for bad in (np.nan, np.inf, -np.inf):
        v = vol.copy()
        v[7, 8, 9] = bad
        for x in (v, _cuda(v)):
            with pytest.raises(ValueError, match="NaN or"):
                inf.log_images(x, 1.0, spacing=SPACING)
        with pytest.raises(ValueError, match="NaN or"):
            inf.log_features(v, mask, 1.0, spacing=SPACING)


def test_abi_refuses_overlaps(inf):
    import torch
    vol = _cuda(np.zeros((6, 6, 6), np.int16))
    w = torch.empty((3, 6, 6, 6), dtype=torch.float64, device="cuda:0")
    out = torch.empty((6, 6, 6), dtype=torch.float64, device="cuda:0")
    eng = inf.engine
    ok = (w[0].data_ptr(), w[1].data_ptr())
    eng.laplacian_of_gaussian_dev(vol.data_ptr(), 0, (6, 6, 6), (1, 1, 1), 1.0, ok, out.data_ptr())
    for works, o in (((w[0].data_ptr(), w[0].data_ptr()), out.data_ptr()),
                     (ok, w[1].data_ptr()),
                     ((w[0].data_ptr() + 8, w[1].data_ptr()), w[0].data_ptr()),
                     ((vol.data_ptr(), w[1].data_ptr()), out.data_ptr())):
        with pytest.raises(ValueError, match="overlaps"):
            eng.laplacian_of_gaussian_dev(vol.data_ptr(), 0, (6, 6, 6), (1, 1, 1), 1.0, works, o)


# ---- features

def same_first_order(got, want, what):
    """FirstOrderFeatures of a float64 image: the histograms and order statistics exactly, the sums (order-dependent in
    the last bits on the float path) within 1e-12 of the feature or of its natural scale."""
    from lungmask_b200 import first_order as fo
    assert [r.label for r in got.rows] == [r.label for r in want.rows], what
    for g, w in zip(got.rows, want.rows):
        assert (g.voxels, g.exact, g.low, g.n_levels) == (w.voxels, w.exact, w.low, w.n_levels), (what, g.label)
        assert np.array_equal(g.histogram, w.histogram) and g.percentiles == w.percentiles, (what, g.label)
        if not w.voxels:
            assert all(math.isnan(x) for x in g.features.values()), (what, g.label)
            continue
        R = max(abs(w.features["Minimum"]), abs(w.features["Maximum"]))
        scale = {"Mean": R, "MeanAbsoluteDeviation": R, "RobustMeanAbsoluteDeviation": R, "RootMeanSquared": R,
                 "Variance": R * R, "Skewness": 1.0, "Kurtosis": 1.0}
        for k in fo.FIRST_ORDER_FEATURES:
            a, b = g.features[k], w.features[k]
            if k in ("Minimum", "Maximum", "Range", "Median", "10Percentile", "90Percentile", "InterquartileRange",
                     "Entropy", "Uniformity") or math.isnan(b):
                assert a == b or (math.isnan(a) and math.isnan(b)), (what, g.label, k)
            else:
                assert abs(a - b) <= 1e-12 * max(abs(b), scale.get(k, 0.0)), (what, g.label, k, a, b)


def check_features(inf, vol, mask, sigmas, bw=25, classes=lg.FEATURE_CLASSES, spacing=SPACING, **settings):
    from lungmask_b200 import texture as tx
    res = inf.log_features(vol, mask, sigmas, bin_width=bw, classes=classes, spacing=spacing, **settings)
    widths = lg.check_bin_widths(bw, lg.check_sigmas(sigmas))
    first, texture_classes = lg.check_classes(classes)
    st = tx.check_settings(settings.get("distances", (1,)), settings.get("force2d", False),
                           settings.get("force2d_dimension", 0), settings.get("weighting_norm"))
    assert [d.name for d in res.images] == list(widths)
    tm = _cuda(mask)
    for s in lg.check_sigmas(sigmas):
        name = lg.image_name(s)
        d = res[name]
        assert d.bin_width == widths[name]
        tb = _cuda(lg.log_host(vol, s, spacing))
        if texture_classes:
            want = inf.texture(tb, tm, widths[name], spacing, texture_classes, 0, st.distances,
                               st.force2d_dimension is not None, st.force2d_dimension or 0, st.weighting_norm)
            assert json.dumps(d.texture.to_dict()) == json.dumps(want.to_dict()), name
        else:
            assert d.texture is None
        if first:
            same_first_order(d.first_order, inf.first_order(tb, tm, widths[name], spacing, 0), name)
        else:
            assert d.first_order is None
    return res


def test_features_two_lungs_and_five_lobes(inf):
    vol = synth.phantom(24, 56, 64, seed=41)
    lungs = two_lungs(*vol.shape)
    res = check_features(inf, vol, lungs, (1.0, 3.0), bw=5)
    assert [r.label for r in res[1.0].first_order.rows] == [1, 2, "lung"]
    v = res.vector("lung")
    assert len(v) == 2 * 91 and list(v)[0] == "log-sigma-1-0-mm-3D_firstorder_10Percentile"
    assert "log-sigma-3-0-mm-3D_glcm_Contrast" in v
    check_features(inf, vol, five_lobes(lungs), (2.0,), bw={2.0: 6}, classes=("glcm", "ngtdm", "firstorder"))
    check_features(inf, vol, lungs, [1.5], bw=5, classes=("glcm", "glrlm"), distances=(1, 2), force2d=True,
                   weighting_norm="euclidean")


def test_features_cuda_inputs_unchanged(inf):
    import torch
    vol = synth.phantom(20, 40, 44, seed=42)
    mask = five_lobes(two_lungs(*vol.shape))
    tv, tm = _cuda(vol), _cuda(mask)
    a = inf.log_features(tv, tm, (1.0, 2.0), bin_width=5, classes=("firstorder", "glszm"), spacing=SPACING)
    b = inf.log_features(vol, mask, (1.0, 2.0), bin_width=5, classes=("firstorder", "glszm"), spacing=SPACING)
    for d, e in zip(a.images, b.images):
        assert json.dumps(d.texture.to_dict()) == json.dumps(e.texture.to_dict()), d.name
        same_first_order(d.first_order, e.first_order, d.name)
    assert a.images[0].first_order.rows[0].voxels > 0
    assert np.array_equal(tv.cpu().numpy(), vol) and torch.equal(tm, _cuda(mask))


# ---- command line

@pytest.mark.parametrize("resample", [False, True])
def test_cli_log_equals_python_chain(tmp_path, resample):
    import torch
    from lungmask_b200 import LMInferer
    from lungmask_b200.__main__ import main
    from lungmask_b200.io import Volume, _write_mha, load_input_image, save_log_features
    p = str(tmp_path / "w.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.mha")
    vol = synth.phantom(12, 96, 96, seed=21)
    _write_mha(src, vol, Volume(vol, (0.7, 0.7, 2.5), (1.0, -2.0, 3.0)))
    J, C = str(tmp_path / "l.json"), str(tmp_path / "l.csv")
    extra = ["--resample", "1,1,1"] if resample else []
    # texture classes only: the first-order sums of a float image are order-dependent in the last bits
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--log", J, "--log-sigma", "1,3",
          "--log-bin-width", "5,3=6", "--log-classes", "glcm,glszm,glrlm,gldm,ngtdm"] + extra)
    main([src, str(tmp_path / "m2.npy"), "--modelpath", p, "--noprogress", "--log", C, "--log-sigma", "1,3",
          "--log-classes", "glcm", "--texture-distances", "1,2"] + extra)
    inferer = LMInferer(modelpath=p, tqdm_disable=True)
    image = load_input_image(src)
    mask = inferer.apply(image)
    if resample:
        r = inferer.resample(image, mask, (1, 1, 1))
        image, mask = r.volume(), r.mask
    J2, C2 = str(tmp_path / "l2.json"), str(tmp_path / "l2.csv")
    save_log_features(J2, inferer.log_features(image, mask, (1, 3), bin_width={1: 5, 3: 6},
                                               classes=("glcm", "glszm", "glrlm", "gldm", "ngtdm")))
    save_log_features(C2, inferer.log_features(image, mask, (1, 3), classes=("glcm",), distances=(1, 2)))
    assert open(J).read() == open(J2).read()
    assert open(C).read() == open(C2).read()
    d = json.loads(open(J).read())
    assert list(d["images"]) == ["log-sigma-1-0-mm-3D", "log-sigma-3-0-mm-3D"]
    assert d["images"]["log-sigma-3-0-mm-3D"]["bin_width"] == 6
    head = open(C).readline().strip().split(",")
    assert head[:3] == ["label", "name", "voxels"] and head[3].startswith("log-sigma-1-0-mm-3D_glcm_")
