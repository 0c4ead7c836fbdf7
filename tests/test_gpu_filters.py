"""PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient image types on the GPU (LMInferer.filtered,
LMInferer.filtered_features; lm_image_range_dev, lm_image_filter_dev, lm_gradient_dev) against the numpy statement
lungmask_b200.filters.filter_host: every image compared as uint64 bit patterns (so -0.0 counts) for every dtype code,
odd and even extents, extents of 1, the table and the arithmetic paths and the 300x512x512 phantom; logarithm and
exponential on the arithmetic path within DESIGN §4.13's ulp bound.  The features of every image type equal `first_order`
and `texture` run on the host-restated image."""
import csv
import json
import math

import numpy as np
import pytest

from lungmask_b200 import _native
from lungmask_b200 import filters as flt
from lungmask_b200 import first_order as fo
from lungmask_b200 import texture as tx
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


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


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


def check_images(got, ref, table, what, spacing=SPACING, names=flt.NAMES):
    """`got` {name: image} against filter_host(ref): bit for bit, except logarithm / exponential off the table path,
    which are within flt.ULP_BOUND with the same sign."""
    assert list(got) == list(names), what
    for name in names:
        want = flt.filter_host(ref, name, spacing=spacing)
        g = got[name].cpu().numpy() if hasattr(got[name], "cpu") else got[name]
        assert g.shape == want.shape and g.dtype == np.float64, (what, name)
        if name in flt.ULP_BOUND and not table:
            assert np.array_equal(np.signbit(g), np.signbit(want)), (what, name)
            worst = float(np.max(ulps(g, want)))
            assert worst <= flt.ULP_BOUND[name], (what, name, worst)
        else:
            assert np.array_equal(bits(g), bits(want)), (what, name)


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
    """u8, i8, i16 and bool take the table, i32 and i64 with their full ranges and every float type the arithmetic."""
    import torch
    shape = (7, 10, 37)
    for k, dtype in enumerate((torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16,
                               torch.bfloat16, torch.float32, torch.float64, torch.bool)):
        t = _values(dtype, shape, 200 + k)
        ref = t.double().numpy()
        table = dtype in (torch.uint8, torch.int8, torch.int16, torch.bool)
        check_images(inf.filtered(t.cuda(), spacing=SPACING), ref, table, (dtype, "cuda"))
        check_images(inf.filtered(t, spacing=SPACING), ref, table, (dtype, "cpu tensor"))


def test_table_and_arithmetic_paths_of_integers(inf):
    """The same int32 / int64 values through the table (max - min < 2^20) and through the arithmetic (one voxel moved
    to widen the range past 2^20)."""
    rng = np.random.default_rng(9)
    for dtype in (np.int32, np.int64):
        v = rng.integers(-1024, 3071, (9, 12, 13)).astype(dtype)
        v.flat[0], v.flat[1] = -1000, 3000
        assert flt.table_span(_native.DTYPE_I32 if dtype == np.int32 else _native.DTYPE_I64, -1024.0, 3071.0)
        check_images(inf.filtered(v, spacing=SPACING), v, True, (dtype, "table"))
        w = v.copy()
        w.flat[2] = 1 << 21
        check_images(inf.filtered(w, spacing=SPACING), w, False, (dtype, "arithmetic"))
        lim = v.astype(np.int64)
        lim.flat[2] = -1024 + (1 << 20) - 1   # max - min = 2^20 - 1: still the table
        check_images(inf.filtered(lim.astype(dtype), spacing=SPACING), lim, True, (dtype, "limit"))


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_images_every_extent_parity_and_one(inf, dtype):
    shapes = [(a, b, c) for a in (1, 2) for b in (1, 3) for c in (1, 4)] + [(5, 6, 7), (33, 17, 70), (2, 64, 1)]
    for i, shape in enumerate(shapes):
        rng = np.random.default_rng(i)
        vol = rng.integers(-1024, 2000, shape).astype(dtype)
        if dtype == np.float32:
            vol = vol + rng.random(shape).astype(np.float32)
        if vol.size == 1:
            vol.flat[0] = 7
        check_images(inf.filtered(vol, spacing=SPACING), vol, dtype == np.int16, (dtype, shape))


def test_images_of_the_300x512x512_phantom(inf):
    """All 5 images of the int16 phantom (the table path), bit for bit; one image on the host at a time."""
    vol = synth.phantom(300, 512, 512, seed=31)
    tv = _cuda(vol)
    for name in flt.NAMES:
        got = inf.filtered(tv, image_types=(name,), spacing=SPACING)[name]
        want = flt.filter_host(vol, name, spacing=SPACING)
        assert np.array_equal(bits(got), bits(want)), name
        del got, want
    assert np.array_equal(tv.cpu().numpy(), vol)


# ---- input kinds and streams

def test_input_kinds_agree(inf):
    import torch
    from lungmask_b200.io import Volume
    vol = np.random.default_rng(3).integers(-1024, 600, (12, 20, 22)).astype(np.int16)
    keep = vol.copy()
    from_np = inf.filtered(vol, spacing=(1.0, 1.0, 2.0))
    from_cpu = inf.filtered(torch.from_numpy(vol), spacing=(1.0, 1.0, 2.0))
    t = _cuda(vol)
    from_cuda = inf.filtered(t, spacing=(1.0, 1.0, 2.0))
    from_volume = inf.filtered(Volume(vol, spacing=(1.0, 1.0, 2.0)))   # the Volume supplies the gradient's spacing
    assert np.array_equal(vol, keep) and np.array_equal(t.cpu().numpy(), keep)
    for name in flt.NAMES:
        a = from_np[name]
        assert isinstance(a, np.ndarray) and a.dtype == np.float64
        b, c = from_cpu[name], from_cuda[name]
        assert isinstance(b, torch.Tensor) and b.device.type == "cpu" and b.dtype == torch.float64
        assert c.is_cuda and c.device.index == inf.engine.device and c.dtype == torch.float64
        assert isinstance(from_volume[name], np.ndarray)
        for other in (b, c, from_volume[name]):
            assert np.array_equal(bits(a), bits(other)), name
    assert len({from_cuda[n].data_ptr() for n in flt.NAMES}) == 5
    unit = inf.filtered(vol, image_types=("gradient",), gradient_use_spacing=False)["gradient"]
    assert np.array_equal(bits(unit), bits(flt.filter_host(vol, "gradient", use_spacing=False)))


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
        got = inf.filtered(t, spacing=SPACING)
        feats = inf.filtered_features(t, m, classes=("firstorder", "glcm"), spacing=SPACING)
    side.synchronize()
    check_images(got, vol, True, "stream")
    want = inf.filtered_features(vol, mask, classes=("firstorder", "glcm"), spacing=SPACING)
    for d, e in zip(feats.images, want.images):   # the float first-order sums are order-dependent in the last bits
        assert json.dumps(d.texture.to_dict()) == json.dumps(e.texture.to_dict()), d.name
        for g, w in zip(d.first_order.rows, e.first_order.rows):
            assert np.array_equal(g.histogram, w.histogram) and g.percentiles == w.percentiles, (d.name, g.label)


# ---- refusals, before any feature kernel

def _count_feature_calls(inf, monkeypatch):
    calls = []
    for fn in ("first_order_sums_dev", "texture_levels_dev", "glcm_dev"):
        orig = getattr(inf.engine, fn)
        monkeypatch.setattr(inf.engine, fn, lambda *a, _f=orig, _n=fn, **k: (calls.append(_n), _f(*a, **k))[1])
    return calls


def test_refusals_before_any_feature_kernel(inf, monkeypatch):
    calls = _count_feature_calls(inf, monkeypatch)
    vol = np.random.default_rng(4).standard_normal((8, 9, 10)).astype(np.float32)
    mask = (np.abs(vol) < 1).astype(np.uint8)
    for bad in (np.nan, np.inf, -np.inf):
        v = vol.copy()
        v[7, 8, 9] = bad
        for x in (v, _cuda(v)):
            for types in (("square",), ("gradient",)):
                with pytest.raises(ValueError, match="NaN or"):
                    inf.filtered(x, image_types=types, spacing=SPACING)
        with pytest.raises(ValueError, match="NaN or"):
            inf.filtered_features(v, mask, spacing=SPACING)
    zeros = np.zeros((6, 7, 8), np.int16)
    for name in ("square", "logarithm", "exponential"):
        with pytest.raises(ValueError, match="all zeros"):
            inf.filtered(zeros, image_types=(name,))
        with pytest.raises(ValueError, match="all zeros"):
            inf.filtered_features(zeros, np.ones(zeros.shape, np.uint8), image_types=("squareroot", name))
    assert not inf.filtered(zeros, image_types=("squareroot",))["squareroot"].any()
    with pytest.raises(ValueError, match="spacing is needed"):
        inf.filtered(vol, image_types=("gradient",))
    with pytest.raises(ValueError, match="spacing is needed"):
        inf.filtered_features(vol, mask)
    with pytest.raises(ValueError, match="unknown image type"):
        inf.filtered(vol, image_types=("lbp2d",))
    with pytest.raises(ValueError, match="unknown feature class"):
        inf.filtered_features(vol, mask, classes=("glcm", "shape"), spacing=SPACING)
    # a ramp that needs far more than 255 levels at bin width 1 in the gradient image only
    shape = (10, 24, 26)
    ramp = np.broadcast_to(np.linspace(-1000.0, 4000.0, shape[2]) ** 2 / 4000.0, shape).astype(np.int16)
    lungs = two_lungs(*shape)
    widths = {n: 1000 for n in flt.NAMES}
    widths["gradient"] = 1
    with pytest.raises(ValueError, match=r"gradient row .* bin width \((\d+) or more\)") as ex:
        inf.filtered_features(ramp, lungs, bin_width=widths, classes=("firstorder", "glcm"), spacing=SPACING)
    assert calls == []
    widths["gradient"] = int(str(ex.value).rsplit("(", 1)[1].split()[0])
    res = inf.filtered_features(ramp, lungs, bin_width=widths, classes=("firstorder", "glcm"), spacing=SPACING)
    assert calls and res["gradient"].bin_width == widths["gradient"] and res["square"].bin_width == 1000


# ---- features

def check_features(inf, vol, mask, bw=25, classes=("firstorder",) + ALL_TEXTURE, alpha=0, shift=0, spacing=SPACING,
                   image_types=None):
    res = inf.filtered_features(vol, mask, image_types=image_types, bin_width=bw, classes=classes, gldm_alpha=alpha,
                                spacing=spacing, voxel_array_shift=shift)
    names = flt.check_image_types(image_types)
    widths = flt.check_bin_widths(bw, names)
    first, texture_classes = flt.check_classes(classes)
    assert [d.name for d in res.images] == list(names)
    tm = _cuda(mask)
    for name in names:
        d = res[name]
        assert d.bin_width == widths[name]
        tb = _cuda(flt.filter_host(vol, name, spacing=spacing))
        if texture_classes:
            want = inf.texture(tb, tm, widths[name], spacing, texture_classes, alpha)
            assert json.dumps(d.texture.to_dict()) == json.dumps(want.to_dict()), name
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
    assert [r.label for r in res["square"].first_order.rows] == [1, 2, "lung"]
    v = res.vector("lung")
    assert len(v) == 5 * 91 and list(v)[0] == "square_firstorder_10Percentile" and "gradient_glcm_Contrast" in v
    check_features(inf, vol, five_lobes(lungs), bw=20, classes=("glcm", "ngtdm", "firstorder"), alpha=2, shift=1024)


def test_features_forty_labels_cuda_inputs_and_subsets(inf):
    import torch
    vol = synth.phantom(20, 40, 44, seed=42)
    rng = np.random.default_rng(43)
    mask = rng.integers(0, 41, vol.shape).astype(np.uint8)
    check_features(inf, vol, mask, bw=40, classes=("firstorder", "glszm", "glrlm", "gldm"),
                   image_types=("logarithm", "gradient"))
    tv, tm = _cuda(vol), _cuda(mask)
    a = inf.filtered_features(tv, tm, bin_width=40, classes=("firstorder", "glcm"), spacing=SPACING)
    b = inf.filtered_features(vol, mask, bin_width=40, classes=("firstorder", "glcm"), spacing=SPACING)
    for d, e in zip(a.images, b.images):
        assert json.dumps(d.texture.to_dict()) == json.dumps(e.texture.to_dict())
    assert np.array_equal(tv.cpu().numpy(), vol) and np.array_equal(tm.cpu().numpy(), mask)
    assert torch.equal(tm, _cuda(mask))


# ---- command line

def test_cli_round_trip(tmp_path):
    import torch
    from lungmask_b200.__main__ import main
    p = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.npy")
    np.save(src, synth.phantom(8, 96, 96, seed=21))
    js, cs = str(tmp_path / "f.json"), str(tmp_path / "f.csv")
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--filtered", js, "--filtered-bin-width",
          "25,gradient=60", "--filtered-classes", "firstorder,glcm"])
    main([src, str(tmp_path / "m2.npy"), "--modelpath", p, "--noprogress", "--filtered", cs, "--filtered-types",
          "square,gradient", "--filtered-classes", "ngtdm"])
    d = json.loads(open(js).read())
    assert d["classes"] == ["firstorder", "glcm"] and d["gradient_use_spacing"] is True
    assert list(d["images"]) == list(flt.NAMES)
    assert d["images"]["gradient"]["bin_width"] == 60 and d["images"]["square"]["bin_width"] == 25
    assert d["images"]["logarithm"]["firstorder"]["rows"][-1]["label"] == "lung"
    lines = list(csv.reader(open(cs)))
    assert lines[0][:3] == ["label", "name", "voxels"]
    assert lines[0][3:] == ["%s_ngtdm_%s" % (n, k) for n in ("square", "gradient") for k in tx.NGTDM_FEATURES]
    assert lines[-1][0] == "lung"
