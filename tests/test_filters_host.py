"""The numpy statement of PyRadiomics' Square, SquareRoot, Logarithm, Exponential and Gradient image types
(lungmask_b200.filters, DESIGN §4.13) on the host: each against a per-voxel restatement of PyRadiomics' code, the
gradient against np.gradient, the integer tables bit for bit against the full-array statement, the refusals, the vector
keys, the writers and the command-line checks."""
import csv
import json
import math

import numpy as np
import pytest

from lungmask_b200 import _native
from lungmask_b200 import filters as flt
from lungmask_b200 import first_order as fo
from lungmask_b200 import texture as tx


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def ulps(a, b):
    """Per-element distance in float64 units in the last place (same-sign finite values)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def sample(seed, shape=(5, 6, 7), scale=900.0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(shape) * scale
    v.flat[:6] = [0.0, -0.0, 1.0, -1.0, 0.5, -0.5]
    return v


# ---- the elementwise types against a per-voxel restatement of PyRadiomics' code

def per_voxel(v, name):
    m = max(abs(float(x)) for x in v.flat)
    out = np.empty(v.shape, np.float64)
    for i, x in enumerate(v.flat):
        x = float(x)
        if name == "square":
            t = (1.0 / math.sqrt(m)) * x
            y = t * t
        elif name == "squareroot":
            y = math.sqrt(x * m) if x > 0 else -math.sqrt(-x * m) if x < 0 else x
        elif name == "logarithm":
            y = math.log(x + 1) if x > 0 else -math.log(-(x - 1)) if x < 0 else x
            y = y * (m / math.log(m + 1))
        else:
            y = math.exp((math.log(m) / m) * x)
        out.flat[i] = y
    return out


@pytest.mark.parametrize("name", flt.ELEMENTWISE)
def test_elementwise_statement_per_voxel(name):
    for seed, scale in ((1, 900.0), (2, 1.0), (3, 3e5)):
        v = sample(seed, scale=scale)
        got = flt.filter_host(v, name)
        want = per_voxel(v, name)
        if name in ("square", "squareroot"):   # correctly rounded operations only: bit for bit
            assert np.array_equal(bits(got), bits(want)), (name, seed)
        else:   # numpy's log / exp against the C library's: a few ulp
            assert np.all(ulps(got, want) <= 4), (name, seed)
            assert np.array_equal(np.signbit(got), np.signbit(want))


def test_zero_signs_and_fixed_points():
    v = np.array([[[0.0, -0.0, 4.0, -4.0, 1.0]]])
    sr = flt.filter_host(v, "squareroot")
    assert bits(sr).ravel().tolist() == bits([0.0, -0.0, 4.0, -4.0, 2.0]).tolist()
    lg = flt.filter_host(v, "logarithm")
    assert bits(lg[0, 0, :2]).tolist() == bits([0.0, -0.0]).tolist()
    assert lg[0, 0, 2] == 4.0 and lg[0, 0, 3] == -4.0   # |x| = m maps to +-m
    sq = flt.filter_host(v, "square")
    assert bits(sq[0, 0, :2]).tolist() == bits([0.0, 0.0]).tolist() and sq[0, 0, 2] == 4.0
    ex = flt.filter_host(v, "exponential")
    assert ex[0, 0, 0] == ex[0, 0, 1] == 1.0 and ex[0, 0, 2] == pytest.approx(4.0, rel=1e-15)
    assert flt.filter_host(np.zeros((2, 2, 2), np.int16), "squareroot").tolist() == np.zeros((2, 2, 2)).tolist()


def test_scalars_are_numpys():
    for m in (1.0, 3.0, 1024.0, 3071.0, 1e-3, 12345.678):
        mm = np.float64(m)
        assert flt.scalar("square", m) == 1 / np.sqrt(mm)
        assert flt.scalar("squareroot", m) == m
        assert flt.scalar("logarithm", m) == mm / np.log(mm + 1)
        assert flt.scalar("exponential", m) == np.log(mm) / mm
        v = np.array([[[-m, 0.5 * m, m]]])
        # the Logarithm scale m / log(m + 1) is the statement's m / max|y|
        y = np.log(np.abs(v) + 1)
        assert mm / np.max(y) == flt.scalar("logarithm", m)


# ---- gradient

def test_gradient_against_np_gradient():
    rng = np.random.default_rng(5)
    v = rng.standard_normal((6, 7, 9)) * 100
    sp = (0.7, 0.8, 2.5)   # (x, y, z)
    got = flt.filter_host(v, "gradient", spacing=sp)
    a = np.zeros(v.shape)
    for s, axis in zip(sp, (2, 1, 0)):
        g = np.gradient(v, s, axis=axis)
        edge = [slice(None)] * 3
        for e in (0, -1):   # ITK's clamped central difference is half of numpy's one-sided one at the edges
            edge[axis] = e
            g[tuple(edge)] *= 0.5
        a += g * g
    assert np.allclose(got, np.sqrt(a), rtol=1e-13, atol=1e-12)
    inner = (slice(1, -1),) * 3
    assert np.allclose(got[inner], np.sqrt(sum(np.gradient(v, s, axis=ax) ** 2
                                                for s, ax in zip(sp, (2, 1, 0))))[inner], rtol=1e-13)


def test_gradient_statement_literal_and_extents_of_one():
    rng = np.random.default_rng(6)
    for shape in ((1, 1, 1), (1, 4, 5), (3, 1, 5), (4, 3, 1), (2, 2, 2)):
        v = rng.integers(-1000, 1000, shape).astype(np.int16)
        sp = (0.703125, 0.9, 1.25)
        got = flt.filter_host(v, "gradient", spacing=sp)
        want = np.empty(shape)
        f = v.astype(np.float64)
        for z in range(shape[0]):
            for y in range(shape[1]):
                for x in range(shape[2]):
                    a = 0.0
                    for s, d in zip(sp, ((0, 0, 1), (0, 1, 0), (1, 0, 0))):
                        inv = 1.0 / s
                        k0, k1, k2 = -0.5 * inv, 0.0 * inv, 0.5 * inv
                        lo = tuple(max(c - o, 0) for c, o in zip((z, y, x), d))
                        hi = tuple(min(c + o, n - 1) for c, o, n in zip((z, y, x), d, shape))
                        g = ((0.0 + k0 * f[lo]) + k1 * f[z, y, x]) + k2 * f[hi]
                        a = a + g * g
                    want[z, y, x] = math.sqrt(a)
        assert np.array_equal(bits(got), bits(want)), shape
    assert not flt.filter_host(np.full((1, 1, 4), 7, np.int16), "gradient", spacing=(1, 1, 1)).any()
    one = flt.filter_host(np.arange(4.0).reshape(1, 1, 4), "gradient", use_spacing=False)
    assert one.tolist() == [[[0.5, 1.0, 1.0, 0.5]]]


# ---- integer tables

@pytest.mark.parametrize("dtype", [np.uint8, np.int8, np.int16, np.int32, np.int64])
def test_table_path_is_the_statement(dtype):
    rng = np.random.default_rng(7)
    info = np.iinfo(dtype)
    lo, hi = max(int(info.min), -3000), min(int(info.max), 5000)
    v = rng.integers(lo, hi + 1, (6, 7, 8)).astype(dtype)
    v.flat[0], v.flat[1] = lo, hi
    code = {np.uint8: _native.DTYPE_U8, np.int8: _native.DTYPE_I8, np.int16: _native.DTYPE_I16,
            np.int32: _native.DTYPE_I32, np.int64: _native.DTYPE_I64}[dtype]
    span = flt.table_span(code, float(v.min()), float(v.max()))
    assert span == (lo, hi - lo + 1)
    for name in flt.ELEMENTWISE:
        t = flt.table(name, *span)
        assert np.array_equal(bits(t[v.astype(np.int64) - span[0]]), bits(flt.filter_host(v, name))), (dtype, name)


def test_table_at_the_span_limit():
    rng = np.random.default_rng(8)
    lo = -(1 << 19) - 12
    hi = lo + (1 << 20) - 1
    v = rng.integers(lo, hi + 1, (4, 16, 16)).astype(np.int32)
    v.flat[0], v.flat[1] = lo, hi
    span = flt.table_span(_native.DTYPE_I32, float(lo), float(hi))
    assert span == (lo, 1 << 20)
    for name in flt.ELEMENTWISE:
        t = flt.table(name, *span)
        assert t.nbytes == 8 << 20
        assert np.array_equal(bits(t[v.astype(np.int64) - lo]), bits(flt.filter_host(v, name))), name
    assert flt.table_span(_native.DTYPE_I32, float(lo), float(hi + 1)) is None
    assert flt.table_span(_native.DTYPE_I64, 0.0, 2.0 ** 53) is None
    assert flt.table_span(_native.DTYPE_F32, 0.0, 10.0) is None


# ---- refusals and argument checks

def test_refusals():
    z = np.zeros((3, 4, 5), np.int16)
    for name in ("square", "logarithm", "exponential"):
        with pytest.raises(ValueError, match="all zeros"):
            flt.filter_host(z, name)
    for bad in (np.nan, np.inf, -np.inf):
        v = np.ones((3, 4, 5))
        v[2, 3, 4] = bad
        for name in flt.NAMES:
            with pytest.raises(ValueError, match="NaN or"):
                flt.filter_host(v, name, spacing=(1, 1, 1))
    with pytest.raises(ValueError, match="spacing is needed"):
        flt.filter_host(z, "gradient")
    for sp in ((1, 1), (1, 0, 1), (1, float("nan"), 1)):
        with pytest.raises(ValueError, match="finite positive"):
            flt.filter_host(z, "gradient", spacing=sp)
    with pytest.raises(ValueError, match="unknown image type"):
        flt.filter_host(z, "lbp3d")
    with pytest.raises(ValueError, match="unknown image type"):
        flt.check_image_types(["square", "log"])
    with pytest.raises(TypeError):
        flt.check_image_types("square")
    with pytest.raises(ValueError):
        flt.check_image_types([])
    assert flt.check_image_types(["gradient", "square"]) == ("square", "gradient")
    assert flt.check_image_types(None) == flt.NAMES
    with pytest.raises(ValueError, match="2\\^32"):
        flt.check_shape((1024, 2048, 2048))
    with pytest.raises(ValueError, match="slices, H, W"):
        flt.check_shape((8, 8))


def test_bin_widths():
    assert flt.check_bin_widths(10) == {n: 10 for n in flt.NAMES}
    assert flt.check_bin_widths(10, ("gradient",)) == {"gradient": 10}
    assert flt.check_bin_widths({"square": 5, "gradient": 7}, ("gradient",)) == {"gradient": 7}
    with pytest.raises(ValueError, match="no bin width for square"):
        flt.check_bin_widths({"gradient": 7}, ("square", "gradient"))
    with pytest.raises(ValueError, match="unknown image type"):
        flt.check_bin_widths({"lbp2d": 7})
    with pytest.raises(ValueError, match="positive"):
        flt.check_bin_widths(0)
    assert flt.parse_bin_widths("25") == {n: 25 for n in flt.NAMES}
    assert flt.parse_bin_widths("25,gradient=10") == dict({n: 25 for n in flt.NAMES}, gradient=10)
    assert flt.parse_bin_widths("gradient=10") == {"gradient": 10}
    for bad in ("", "x", "25,grad=3", "25,square=a", "25,30", "0", "25,square=0"):
        with pytest.raises((TypeError, ValueError)):
            flt.parse_bin_widths(bad)


# ---- result, writers and command line

def synthetic_features(classes=flt.FEATURE_CLASSES, seed=0):
    """A FilteredFeatures built on the host for two rows (label 1 and "lung") of a tiny volume: first-order rows from
    first_order.sums_host and texture rows from random exact matrices."""
    rng = np.random.default_rng(seed)
    vol = rng.integers(-900, -600, (6, 6, 6)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    mask[1:5, 1:5, 1:5] = 1
    first, texture_classes = flt.check_classes(classes)
    images = []
    for name in flt.NAMES:
        image = flt.filter_host(vol, name, spacing=(1.0, 1.0, 2.0))
        bw = 10 if name == "gradient" else 25
        d = flt.ImageFeatures(name, bw)
        v = image[mask > 0]
        if first:
            rows = []
            for r in (1, 256):
                plan = fo.plan_row(v.size, float(v.min()), float(v.max()), float(np.mean(v)),
                                   np.percentile(v, fo.PERCENTILES), bw, False)
                rows.append(fo.build_row(r, "lung" if r == 256 else "left", bw, plan, *fo.sums_host(v, plan, bw),
                                         spacing=(1.0, 1.0, 2.0)))
            d.first_order = fo.FirstOrderFeatures((1.0, 1.0, 2.0), bw, 0, rows)
        if texture_classes:
            low, ng = tx.discretisation(float(v.min()), float(v.max()), bw)
            rows = []
            for r in (1, 256):
                U = rng.integers(0, 5, (13, ng * (ng + 1) // 2))
                zones = np.array([[1, 2, 3]], np.int64)
                runs = rng.integers(0, 3, (13, ng, 6))
                G, N, A = (rng.integers(0, 4, (ng, 27)) for _ in range(3))
                rows.append(tx.build_row(r, "lung" if r == 256 else "left", v.size, bw, low, ng, U, zones,
                                         texture_classes, runs, (G, N, A)))
            d.texture = tx.TextureFeatures((1.0, 1.0, 2.0), bw, rows, texture_classes, 0)
        images.append(d)
    computed = (("firstorder",) if first else ()) + texture_classes
    return flt.FilteredFeatures(computed, (1.0, 1.0, 2.0), 0, 0, True, images)


def test_vector_keys_follow_image_class_and_feature_order():
    f = synthetic_features()
    keys = list(f.vector(1))
    names = (fo.FIRST_ORDER_FEATURES, tx.GLCM_FEATURES, tx.GLSZM_FEATURES, tx.GLRLM_FEATURES, tx.GLDM_FEATURES,
             tx.NGTDM_FEATURES)
    want = ["%s_%s_%s" % (d, c, k) for d in flt.NAMES for c, ks in zip(flt.FEATURE_CLASSES, names) for k in ks]
    assert keys == want and len(keys) == 5 * 91
    assert keys[0] == "square_firstorder_10Percentile" and "gradient_glcm_Contrast" in keys
    assert f["gradient"].bin_width == 10
    v = f.vector("lung")
    assert v["logarithm_firstorder_Mean"] == f["logarithm"].first_order["lung"].features["Mean"]
    assert v["exponential_ngtdm_Busyness"] == f["exponential"].texture["lung"].ngtdm["Busyness"]
    sub = synthetic_features(("glrlm", "firstorder"))
    assert sub.classes == ("firstorder", "glrlm")
    assert all(k.split("_")[1] in ("firstorder", "glrlm") for k in sub.vector(1))


def test_writers_round_trip(tmp_path):
    from lungmask_b200.io import save_filtered_features
    f = synthetic_features()
    save_filtered_features(str(tmp_path / "f.json"), f)
    d = json.loads((tmp_path / "f.json").read_text())
    assert d == json.loads(json.dumps(f.to_dict()))
    assert list(d["images"]) == list(flt.NAMES) and d["images"]["gradient"]["bin_width"] == 10
    assert d["images"]["square"]["texture"] == json.loads(json.dumps(f["square"].texture.to_dict()))
    save_filtered_features(str(tmp_path / "f.csv"), f)
    with open(tmp_path / "f.csv") as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["label", "name", "voxels"] + list(f.vector(1))
    assert [r[:3] for r in rows[1:]] == [["1", "left", "64"], ["lung", "lung", "64"]]
    for r, label in zip(rows[1:], (1, "lung")):
        want = f.vector(label)
        for k, cell in zip(rows[0][3:], r[3:]):
            assert float(cell) == want[k] or (math.isnan(float(cell)) and math.isnan(want[k])), k
    with pytest.raises(SystemExit):
        save_filtered_features(str(tmp_path / "f.txt"), f)


def test_cli_flags_and_checks_before_segmentation(tmp_path):
    from lungmask_b200.__main__ import build_parser, main
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    a = build_parser().parse_args([str(inp), "out.npy"])
    assert (a.filtered, a.filtered_bin_width) == (None, "25")
    assert a.filtered_types == "square,squareroot,logarithm,exponential,gradient"
    assert a.filtered_classes == "firstorder,glcm,glszm,glrlm,gldm,ngtdm"
    a = build_parser().parse_args([str(inp), "out.npy", "--filtered", "f.csv", "--filtered-types", "square,gradient",
                                   "--filtered-bin-width", "25,gradient=10", "--filtered-classes", "firstorder,glcm"])
    assert (a.filtered, a.filtered_types, a.filtered_bin_width, a.filtered_classes) == (
        "f.csv", "square,gradient", "25,gradient=10", "firstorder,glcm")
    out = str(tmp_path / "m.npy")
    # every check ends the run before the volume is segmented (that would need a model and a GPU)
    for extra, msg in (((), "unsupported filtered output"),
                       (("--filtered-types", "square,lbp3d"), "filtered-types"),
                       (("--filtered-types", ","), "filtered-types"),
                       (("--filtered-bin-width", "0"), "filtered-bin-width"),
                       (("--filtered-bin-width", "25,grad=3"), "filtered-bin-width"),
                       (("--filtered-types", "gradient", "--filtered-bin-width", "square=10"), "filtered-bin-width"),
                       (("--filtered-classes", "glcm,shape"), "filtered-classes")):
        path = str(tmp_path / ("f.xlsx" if not extra else "f.json"))
        with pytest.raises(SystemExit, match=msg):
            main([str(inp), out, "--filtered", path, *extra])
