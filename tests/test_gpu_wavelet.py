"""Wavelet decompositions on the GPU (LMInferer.wavelet, LMInferer.wavelet_features, lm_wavelet_dev) against the numpy
statement lungmask_b200.wavelet.swt_host: every band bit for bit (uint64 patterns, so -0.0 counts) for every dtype code,
odd and even extents and the 300x512x512 phantom; and the features of every decomposition equal to `first_order` and
`texture` run on the host-restated band."""
import csv
import json
import math

import numpy as np
import pytest

from lungmask_b200 import first_order as fo
from lungmask_b200 import texture as tx
from lungmask_b200 import wavelet as wv
from oracle import synth

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 2.5)   # (x, y, z) mm
ALL_TEXTURE = tx.CLASSES


@pytest.fixture(scope="module")
def inf():
    import os
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=53, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def bits(a):
    import torch
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


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


def random_labels(seed, shape, labels):
    import scipy.ndimage as ndi
    rng = np.random.default_rng(seed)
    field = ndi.gaussian_filter(rng.standard_normal(shape), 1.5)
    m = (field > np.quantile(field, 0.4)).astype(np.uint8)
    region = ndi.gaussian_filter(rng.standard_normal(shape), 2.5)
    cuts = np.quantile(region, np.linspace(0, 1, labels + 1)[1:-1])
    return m * (np.searchsorted(cuts, region) + 1).astype(np.uint8)


def check_bands(got, want, what):
    assert list(got) == list(want), what
    for name in want:
        assert tuple(got[name].shape) == want[name].shape, (what, name)
        assert np.array_equal(bits(got[name]), bits(want[name])), (what, name)


# ---- bands

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


def test_bands_every_dtype_code(inf):
    import torch
    shape = (7, 10, 37)
    for k, dtype in enumerate((torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16, torch.bfloat16,
                               torch.float32, torch.float64, torch.bool)):
        t = _values(dtype, shape, 100 + k)
        ref = t.double().numpy()
        for wavelet in wv.WAVELETS:
            want = wv.swt_host(ref, wavelet)
            check_bands(inf.wavelet(t.cuda(), wavelet), want, (dtype, wavelet, "cuda"))
            check_bands(inf.wavelet(t, wavelet), want, (dtype, wavelet, "cpu tensor"))


@pytest.mark.parametrize("wavelet,shapes", [
    ("coif1", [(a, b, c) for a in (5, 6) for b in (5, 6) for c in (5, 6)] + [(9, 17, 70), (33, 40, 5)]),
    ("haar", [(a, b, c) for a in (1, 2) for b in (1, 2) for c in (1, 2)] + [(3, 31, 66), (40, 1, 3)]),
])
def test_bands_every_extent_parity(inf, wavelet, shapes):
    for i, shape in enumerate(shapes):
        vol = np.random.default_rng(i).integers(-1024, 2000, shape).astype(np.int16)
        check_bands(inf.wavelet(vol, wavelet), wv.swt_host(vol, wavelet), (wavelet, shape))


def test_bands_of_the_300x512x512_phantom(inf):
    """All 8 coif1 bands of the int16 phantom; the host reference shares its x and y passes between the bands."""
    vol = synth.phantom(300, 512, 512, seed=31)
    tv = _cuda(vol)
    lo, hi = wv.decomposition_filters("coif1")
    v = vol.astype(np.float64)
    for hx in (0, 1):
        X = wv.swt_pass(v, (lo, hi)[hx], 2)
        for hy in (0, 1):
            Y = wv.swt_pass(X, (lo, hi)[hy], 1)
            for hz in (0, 1):
                name = "wavelet-" + "LH"[hx] + "LH"[hy] + "LH"[hz]
                want = wv.swt_pass(Y, (lo, hi)[hz], 0)
                got = inf.wavelet(tv, decompositions=(name,))[name]
                assert np.array_equal(bits(got), bits(want)), name
                del got, want
    assert np.array_equal(tv.cpu().numpy(), vol)


# ---- input kinds and refusals

def test_input_kinds_agree(inf):
    import torch
    from lungmask_b200.io import Volume
    vol = np.random.default_rng(3).integers(-1024, 600, (12, 20, 22)).astype(np.int16)
    keep = vol.copy()
    from_np = inf.wavelet(vol)
    from_cpu = inf.wavelet(torch.from_numpy(vol))
    t = _cuda(vol)
    from_cuda = inf.wavelet(t)
    from_volume = inf.wavelet(Volume(vol, spacing=(1.0, 1.0, 2.0)))
    assert np.array_equal(vol, keep) and np.array_equal(t.cpu().numpy(), keep)
    for name in wv.NAMES:
        a = from_np[name]
        assert isinstance(a, np.ndarray) and a.dtype == np.float64
        b, c = from_cpu[name], from_cuda[name]
        assert isinstance(b, torch.Tensor) and b.device.type == "cpu" and b.dtype == torch.float64
        assert c.is_cuda and c.device.index == inf.engine.device and c.dtype == torch.float64
        assert isinstance(from_volume[name], np.ndarray)
        for other in (b, c, from_volume[name]):
            assert np.array_equal(bits(a), bits(other)), name
    assert len({from_cuda[n].data_ptr() for n in wv.NAMES}) == 8


def test_refusals(inf):
    vol = np.random.default_rng(4).standard_normal((8, 9, 10)).astype(np.float32)
    for bad in (np.nan, np.inf, -np.inf):
        v = vol.copy()
        v[7, 8, 9] = bad
        for x in (v, _cuda(v)):
            with pytest.raises(ValueError, match="NaN or"):
                inf.wavelet(x, decompositions=("LLL",))
        with pytest.raises(ValueError, match="NaN or"):
            inf.wavelet_features(v, (np.abs(v) < 1).astype(np.uint8))
    with pytest.raises(ValueError, match="padded extent"):
        inf.wavelet(np.zeros((4, 9, 10), np.int16))
    with pytest.raises(ValueError, match="padded extent"):
        inf.wavelet_features(np.zeros((9, 9, 3), np.int16), np.ones((9, 9, 3), np.uint8))
    with pytest.raises(ValueError, match="unknown wavelet"):
        inf.wavelet(vol, wavelet="db2")
    with pytest.raises(ValueError, match="unknown wavelet"):
        inf.wavelet_features(vol, np.ones(vol.shape, np.uint8), wavelet="sym4")
    with pytest.raises(ValueError, match="unknown feature class"):
        inf.wavelet_features(vol, np.ones(vol.shape, np.uint8), classes=("glcm", "shape"))


# ---- features

def check_features(inf, vol, mask, bw=25, classes=("firstorder",) + ALL_TEXTURE, alpha=0, shift=0, spacing=SPACING):
    res = inf.wavelet_features(vol, mask, bin_width=bw, classes=classes, gldm_alpha=alpha, spacing=spacing,
                               voxel_array_shift=shift)
    widths = wv.check_bin_widths(bw)
    first, texture_classes = wv.check_classes(classes)
    assert [d.name for d in res.decompositions] == list(wv.NAMES)
    tm = _cuda(mask)
    for name, band in wv.swt_host(vol).items():
        d = res[name]
        assert d.bin_width == widths[name]
        tb = _cuda(band)
        if texture_classes:
            want = inf.texture(tb, tm, widths[name], spacing, texture_classes, alpha)
            assert json.dumps(d.texture.to_dict()) == json.dumps(want.to_dict()), name
            for g, w in zip(d.texture.rows, want.rows):
                for c in texture_classes:
                    assert all(a == b or (math.isnan(a) and math.isnan(b))
                               for a, b in zip(getattr(g, c).values(), getattr(w, c).values())), (name, g.label, c)
        else:
            assert d.texture is None
        if first:
            want = inf.first_order(tb, tm, widths[name], spacing, shift)
            assert [r.label for r in d.first_order.rows] == [r.label for r in want.rows]
            for g, w in zip(d.first_order.rows, want.rows):
                assert (g.voxels, g.exact, g.low, g.n_levels) == (w.voxels, w.exact, w.low, w.n_levels), (name, g.label)
                assert np.array_equal(g.histogram, w.histogram) and g.percentiles == w.percentiles, (name, g.label)
                if not w.voxels:
                    assert all(math.isnan(x) for x in g.features.values()), (name, g.label)
                    continue
                # the float path's sums are order-dependent in the last bits: 1e-12 of the feature, or of its natural
                # scale where it can be near zero (R the largest |value|)
                R = max(abs(w.features["Minimum"]), abs(w.features["Maximum"]))
                scale = {"Mean": R, "MeanAbsoluteDeviation": R, "RobustMeanAbsoluteDeviation": R, "RootMeanSquared": R,
                         "Variance": R * R, "Skewness": 1.0, "Kurtosis": 1.0}
                for k in fo.FIRST_ORDER_FEATURES:
                    a, b = g.features[k], w.features[k]
                    if k in ("Minimum", "Maximum", "Range", "Median", "10Percentile", "90Percentile",
                             "InterquartileRange", "Entropy", "Uniformity") or math.isnan(b):
                        assert a == b or (math.isnan(a) and math.isnan(b)), (name, g.label, k)
                    else:
                        assert abs(a - b) <= 1e-12 * max(abs(b), scale.get(k, 0.0)), (name, g.label, k, a, b)
        else:
            assert d.first_order is None
    return res


def test_features_two_lungs_and_five_lobes(inf):
    vol = synth.phantom(24, 56, 64, seed=41)
    lungs = two_lungs(*vol.shape)
    res = check_features(inf, vol, lungs)
    assert [r.label for r in res["LLH"].first_order.rows] == [1, 2, "lung"]
    v = res.vector("lung")
    assert len(v) == 8 * 91 and list(v)[0] == "wavelet-LLH_firstorder_10Percentile"
    check_features(inf, vol, five_lobes(lungs), bw=20, classes=("glcm", "ngtdm", "firstorder"), alpha=2, shift=1024)


def test_features_forty_labels_cuda_inputs(inf):
    import torch
    vol = synth.phantom(20, 40, 44, seed=42)
    mask = random_labels(43, vol.shape, 40)
    assert len(np.unique(mask)) == 41
    check_features(inf, vol, mask, bw=40, classes=("firstorder", "glszm", "glrlm", "gldm"))
    tv, tm = _cuda(vol), _cuda(mask)
    a = inf.wavelet_features(tv, tm, bin_width=40, classes=("firstorder", "glcm"))
    b = inf.wavelet_features(vol, mask, bin_width=40, classes=("firstorder", "glcm"))
    for d, e in zip(a.decompositions, b.decompositions):
        assert json.dumps(d.texture.to_dict()) == json.dumps(e.texture.to_dict())
    assert np.array_equal(tv.cpu().numpy(), vol) and np.array_equal(tm.cpu().numpy(), mask)
    assert a.spacing is None and isinstance(a.decompositions[0].first_order.rows[0].features["Mean"], float)
    assert torch.equal(tm, _cuda(mask))


def test_features_absent_model_label(inf):
    vol = synth.phantom(16, 40, 48, seed=44)
    mask = two_lungs(*vol.shape)
    mask[mask == 2] = 0
    res = check_features(inf, vol, mask, classes=("firstorder", "glcm"))
    for d in res.decompositions:
        assert d.first_order[2].voxels == 0 and all(math.isnan(x) for x in d.first_order[2].features.values())
        assert d.texture[2].voxels == 0 and all(math.isnan(x) for x in d.texture[2].glcm.values())
    assert all(math.isnan(x) for x in res.vector(2).values())


# ---- bin widths

def test_bin_width_per_decomposition_and_the_lll_refusal(inf, monkeypatch):
    rng = np.random.default_rng(45)
    shape = (10, 24, 26)
    ramp = np.broadcast_to(np.linspace(-1000.0, 4000.0, shape[2]), shape)
    vol = (ramp + rng.integers(-20, 20, shape)).astype(np.int16)
    mask = two_lungs(*vol.shape)
    widths = {n: 1000 for n in wv.NAMES}
    widths["wavelet-LLL"] = 25
    # the lungs see about 3300 HU of the ramp, which LLL scales by 2.8: more than 255 levels at 25
    calls = []
    for fn in ("first_order_sums_dev", "texture_levels_dev", "glcm_dev"):
        orig = getattr(inf.engine, fn)
        monkeypatch.setattr(inf.engine, fn, lambda *a, _f=orig, _n=fn, **k: (calls.append(_n), _f(*a, **k))[1])
    with pytest.raises(ValueError, match=r"wavelet-LLL row .* bin width \((\d+) or more\)") as ex:
        inf.wavelet_features(vol, mask, bin_width=widths, classes=("firstorder", "glcm"))
    assert calls == []
    wider = int(str(ex.value).rsplit("(", 1)[1].split()[0])
    widths["wavelet-LLL"] = wider
    res = check_features(inf, vol, mask, bw=widths, classes=("firstorder", "glcm"))
    assert calls and res["LLL"].bin_width == wider and res["LLH"].bin_width == 1000
    assert res["LLL"].first_order.bin_width == wider and res["HHH"].texture.bin_width == 1000


# ---- command line

def test_cli_round_trip(tmp_path):
    import torch
    from lungmask_b200.__main__ import main
    p = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.npy")
    np.save(src, synth.phantom(8, 96, 96, seed=21))
    js, cs = str(tmp_path / "w.json"), str(tmp_path / "w.csv")
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--wavelet", js, "--wavelet-bin-width",
          "25,LLL=60", "--wavelet-classes", "firstorder,glcm"])
    main([src, str(tmp_path / "m2.npy"), "--modelpath", p, "--noprogress", "--wavelet", cs, "--wavelet-name", "haar",
          "--wavelet-classes", "ngtdm"])
    d = json.loads(open(js).read())
    assert d["wavelet"] == "coif1" and d["classes"] == ["firstorder", "glcm"]
    assert list(d["decompositions"]) == list(wv.NAMES)
    assert d["decompositions"]["wavelet-LLL"]["bin_width"] == 60 and d["decompositions"]["wavelet-HHL"]["bin_width"] == 25
    assert d["decompositions"]["wavelet-LLH"]["firstorder"]["rows"][-1]["label"] == "lung"
    lines = list(csv.reader(open(cs)))
    assert lines[0][:3] == ["label", "name", "voxels"]
    assert lines[0][3:] == ["%s_ngtdm_%s" % (n, k) for n in wv.NAMES for k in tx.NGTDM_FEATURES]
    assert lines[-1][0] == "lung"
