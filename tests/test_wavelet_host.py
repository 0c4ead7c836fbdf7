"""The wavelet decomposition's host side (lungmask_b200.wavelet; DESIGN §4.12): the taps against the closed form, swt_host
bit for bit against a brute-force loop with explicit modular indices, known answers, Parseval, shift and linearity, the
names, the argument checks, the writers and the command-line checks."""
import csv
import decimal
import itertools
import json
import math

import numpy as np
import pytest

from lungmask_b200 import first_order as fo
from lungmask_b200 import texture as tx
from lungmask_b200 import wavelet as wv


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


# ---- taps

def coif1_closed_form():
    """Daubechies' coif1 scaling filter at 50 digits: (-3 + r, 1 - r, 14 - 2r, 14 + 2r, 5 + r, 1 - r) / (16 sqrt 2), r = sqrt 7."""
    with decimal.localcontext() as ctx:
        ctx.prec = 50
        r, d = decimal.Decimal(7).sqrt(), 16 * decimal.Decimal(2).sqrt()
        return [x / d for x in (-3 + r, 1 - r, 14 - 2 * r, 14 + 2 * r, 5 + r, 1 - r)]


def test_coif1_taps_match_the_closed_form():
    # relative to the largest tap: PyWavelets' table sits 3e-13..7e-13 from the closed form on every tap (2e-11 of the
    # smallest tap itself), so this catches a transcription error, not the table's offset
    want = coif1_closed_form()
    norm = max(abs(w) for w in want)
    for got, w in zip(wv.DEC_LO["coif1"], want):
        assert abs(decimal.Decimal(got) - w) <= decimal.Decimal("1e-11") * norm, (got, w)


@pytest.mark.parametrize("name", wv.WAVELETS)
def test_taps_are_an_orthonormal_qmf_pair(name):
    lo, hi = wv.decomposition_filters(name)
    F = lo.size
    assert all(hi[k] == (-1) ** (k + 1) * lo[F - 1 - k] for k in range(F))   # exact: a sign flip
    assert abs(math.fsum(lo) - math.sqrt(2)) < 1e-11
    for f in (lo, hi):
        assert abs(math.fsum(f * f) - 1.0) < 1e-11
        for m in range(1, F // 2):
            assert abs(math.fsum(f[k] * f[k + 2 * m] for k in range(F - 2 * m))) < 1e-11
    assert abs(math.fsum(lo * hi)) < 1e-11


# ---- the restatement against a brute-force loop

def brute_force(vol, wavelet):
    """Every band by three explicit loops over the voxels, one per pass, with the modular index of the padded axis."""
    lo, hi = (list(map(float, f)) for f in wv.decomposition_filters(wavelet))
    F = len(lo)
    v = np.asarray(vol).astype(np.float64)

    def index(k, n):
        npad = n + n % 2
        m = k % npad
        return 0 if m == n else m

    def run(a, taps, axis):
        out = np.empty(a.shape, np.float64)
        n = a.shape[axis]
        for pos in itertools.product(*(range(s) for s in a.shape)):
            acc = 0.0
            for j in range(F):
                src = list(pos)
                src[axis] = index(pos[axis] + F // 2 - j, n)
                acc = acc + taps[j] * float(a[tuple(src)])
            out[pos] = acc
        return out

    res = {}
    for name in wv.NAMES:
        hx, hy, hz = (c == "H" for c in name[-3:])
        a = run(v, hi if hx else lo, 2)
        a = run(a, hi if hy else lo, 1)
        res[name] = run(a, hi if hz else lo, 0)
    return res


def _inputs(shape, seed):
    rng = np.random.default_rng(seed)
    signed_zero = np.where(rng.random(shape) < 0.5, -0.0, 0.0)
    mixed = np.where(rng.random(shape) < 0.3, signed_zero, rng.standard_normal(shape) * 300.0)
    return [rng.integers(-1024, 3000, shape).astype(np.int16), (rng.standard_normal(shape) * 1e3).astype(np.float32),
            signed_zero, mixed]


@pytest.mark.parametrize("wavelet,shape", [("coif1", s) for s in itertools.product((5, 6), repeat=3)] +
                         [("coif1", (7, 8, 9))] +
                         [("haar", s) for s in itertools.product((1, 2), repeat=3)] + [("haar", (3, 4, 5))])
def test_swt_host_is_bit_identical_to_a_brute_force_loop(wavelet, shape):
    for k, vol in enumerate(_inputs(shape, 11 + sum(shape))):
        got, want = wv.swt_host(vol, wavelet), brute_force(vol, wavelet)
        assert list(got) == list(wv.NAMES)
        for name in wv.NAMES:
            assert got[name].shape == shape and got[name].dtype == np.float64
            assert np.array_equal(bits(got[name]), bits(want[name])), (wavelet, shape, k, name)


def test_swt_host_decomposition_subset():
    vol = _inputs((6, 7, 8), 3)[0]
    every = wv.swt_host(vol)
    some = wv.swt_host(vol, decompositions=("LLL", "wavelet-HLH"))
    assert list(some) == ["wavelet-HLH", "wavelet-LLL"]
    for name, band in some.items():
        assert np.array_equal(bits(band), bits(every[name]))


# ---- known answers and properties

@pytest.mark.parametrize("axis", [0, 1, 2])
def test_haar_known_answer_along_each_axis(axis):
    shape = [2, 2, 2]
    shape[axis] = 4
    vol = np.moveaxis(np.broadcast_to(np.array([1.0, 2.0, 3.0, 4.0]), shape[:axis] + shape[axis + 1:] + [4]), -1, axis)
    low = np.array([3.0, 5.0, 7.0, 5.0]) / math.sqrt(2)
    high = np.array([-1.0, -1.0, -1.0, 3.0]) / math.sqrt(2)
    res = wv.swt_host(vol, "haar")
    letter = 2 - axis          # the letters are (x, y, z) = axes (2, 1, 0)
    for name, band in res.items():
        code = name[-3:]
        others_low = all(c == "L" for i, c in enumerate(code) if i != letter)
        if not others_low:     # a high-pass along a constant axis
            assert np.all(band == 0), name
            continue
        # the two low-pass passes along the constant axes of extent 2 give sqrt(2)^2 = 2
        want = 2.0 * (high if code[letter] == "H" else low)
        assert np.allclose(np.moveaxis(band, axis, -1), want, rtol=1e-15, atol=1e-15), name


def test_parseval_on_even_extents():
    rng = np.random.default_rng(5)
    for wavelet in wv.WAVELETS:
        vol = rng.standard_normal((6, 8, 10)) * 100.0
        energy = math.fsum(float((b * b).sum()) for b in wv.swt_host(vol, wavelet).values())
        assert abs(energy - 8.0 * float((vol * vol).sum())) <= 1e-10 * energy


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_circular_shift_of_an_even_axis_shifts_every_band(axis):
    vol = _inputs((6, 8, 10), 7)[3]
    base, rolled = wv.swt_host(vol), wv.swt_host(np.roll(vol, 1, axis=axis))
    for name in wv.NAMES:
        assert np.array_equal(bits(np.roll(base[name], 1, axis=axis)), bits(rolled[name])), name


def test_linearity_within_rounding():
    rng = np.random.default_rng(9)
    x, y = rng.standard_normal((2, 7, 6, 5)) * 500.0
    bx, by, bxy = wv.swt_host(x), wv.swt_host(y), wv.swt_host(3.0 * x - y)
    for name in wv.NAMES:
        assert np.allclose(bxy[name], 3.0 * bx[name] - by[name], rtol=0, atol=1e-9), name


# ---- names, order, vector keys

def test_names_order_and_band_codes():
    assert wv.NAMES == ("wavelet-LLH", "wavelet-LHL", "wavelet-LHH", "wavelet-HLL", "wavelet-HLH", "wavelet-HHL",
                        "wavelet-HHH", "wavelet-LLL")
    assert [wv.band_code(n) for n in wv.NAMES] == [1, 2, 3, 4, 5, 6, 7, 0]
    assert wv.decomposition_name("LLH") == wv.decomposition_name("wavelet-LLH") == "wavelet-LLH"
    assert wv.check_decompositions(None) == wv.NAMES
    assert wv.check_decompositions(["wavelet-LLL", "HHH", "LLH"]) == ("wavelet-LLH", "wavelet-HHH", "wavelet-LLL")


def synthetic_features(classes=wv.FEATURE_CLASSES, seed=0):
    """A WaveletFeatures built on the host for two rows (label 1 and "lung") of a tiny volume: first-order rows from
    first_order.sums_host and texture rows from random exact matrices."""
    rng = np.random.default_rng(seed)
    vol = rng.integers(-900, -600, (6, 6, 6)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    mask[1:5, 1:5, 1:5] = 1
    first, texture_classes = wv.check_classes(classes)
    decomps = []
    for name, band in wv.swt_host(vol).items():
        bw = 25 if name != "wavelet-LLL" else 50
        d = wv.WaveletDecomposition(name, bw)
        v = band[mask > 0]
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
        decomps.append(d)
    computed = (("firstorder",) if first else ()) + texture_classes
    return wv.WaveletFeatures("coif1", computed, (1.0, 1.0, 2.0), 0, 0, decomps)


def test_vector_keys_follow_decomposition_class_and_feature_order():
    f = synthetic_features()
    keys = list(f.vector(1))
    names = (fo.FIRST_ORDER_FEATURES, tx.GLCM_FEATURES, tx.GLSZM_FEATURES, tx.GLRLM_FEATURES, tx.GLDM_FEATURES,
             tx.NGTDM_FEATURES)
    want = ["%s_%s_%s" % (d, c, k) for d in wv.NAMES for c, ks in zip(wv.FEATURE_CLASSES, names) for k in ks]
    assert keys == want and len(keys) == 8 * 91
    assert keys[0] == "wavelet-LLH_firstorder_10Percentile" and "wavelet-LLL_glcm_Contrast" in keys
    assert f["LLL"] is f["wavelet-LLL"] and f["LLL"].bin_width == 50
    v = f.vector("lung")
    assert v["wavelet-HLH_firstorder_Mean"] == f["wavelet-HLH"].first_order["lung"].features["Mean"]
    assert v["wavelet-LHL_ngtdm_Busyness"] == f["wavelet-LHL"].texture["lung"].ngtdm["Busyness"]
    sub = synthetic_features(("glrlm", "firstorder"))
    assert sub.classes == ("firstorder", "glrlm")
    assert all(k.split("_")[1] in ("firstorder", "glrlm") for k in sub.vector(1))


# ---- argument errors

def test_argument_errors():
    with pytest.raises(ValueError, match="unknown wavelet"):
        wv.check_wavelet("db2")
    with pytest.raises(TypeError):
        wv.check_wavelet(1)
    assert wv.check_shape((5, 5, 5), "coif1") == (5, 5, 5)
    assert wv.check_shape((6, 1, 6), "haar") == (6, 1, 6)
    for shape in ((4, 8, 8), (8, 3, 8), (8, 8, 2)):
        with pytest.raises(ValueError, match="padded extent"):
            wv.check_shape(shape, "coif1")
    with pytest.raises(ValueError, match="2\\^32"):
        wv.check_shape((1024, 2048, 2048), "coif1")
    with pytest.raises(ValueError, match="slices, H, W"):
        wv.check_shape((8, 8), "coif1")
    with pytest.raises(ValueError, match="padded extent"):
        wv.swt_host(np.zeros((4, 8, 8)), "coif1")
    assert wv.check_bin_widths(10) == {n: 10 for n in wv.NAMES}
    full = {n: 25 for n in wv.NAMES}
    assert wv.check_bin_widths(dict(full, **{"wavelet-LLL": 60}))["wavelet-LLL"] == 60
    with pytest.raises(ValueError, match="no bin width for wavelet-LLL"):
        wv.check_bin_widths({n: 25 for n in wv.NAMES[:-1]})
    with pytest.raises(ValueError, match="unknown wavelet decomposition"):
        wv.check_bin_widths(dict(full, XYZ=3))
    with pytest.raises(ValueError, match="given twice"):
        wv.check_bin_widths(dict(full, LLL=3))
    with pytest.raises(ValueError, match="positive"):
        wv.check_bin_widths({**{n: 25 for n in wv.NAMES[:-1]}, "LLL": 0})
    with pytest.raises(TypeError):
        wv.check_bin_widths(2.5)
    assert wv.check_classes(["ngtdm", "firstorder"]) == (True, ("ngtdm",))
    assert wv.check_classes(["glcm"]) == (False, ("glcm",))
    for bad, exc in (([], ValueError), (["shape"], ValueError), ("glcm", TypeError), ([1], TypeError)):
        with pytest.raises(exc):
            wv.check_classes(bad)
    with pytest.raises(ValueError, match="unknown wavelet decomposition"):
        wv.check_decompositions(["LLX"])
    with pytest.raises(ValueError):
        wv.check_decompositions([])


def test_parse_bin_widths():
    assert wv.parse_bin_widths("25") == {n: 25 for n in wv.NAMES}
    assert wv.parse_bin_widths("25,LLL=50") == dict({n: 25 for n in wv.NAMES}, **{"wavelet-LLL": 50})
    assert wv.parse_bin_widths("30, wavelet-HHH=10,LLH=5")["wavelet-LLH"] == 5
    for bad in ("", "x", "25,LLQ=3", "25,LLL=a", "25,30", "LLL=50", "0"):
        with pytest.raises((TypeError, ValueError)):
            wv.parse_bin_widths(bad)


# ---- writers and command line

def test_writers_round_trip(tmp_path):
    from lungmask_b200.io import save_wavelet_features
    f = synthetic_features()
    save_wavelet_features(str(tmp_path / "w.json"), f)
    d = json.loads((tmp_path / "w.json").read_text())
    assert d == json.loads(json.dumps(f.to_dict()))
    assert list(d["decompositions"]) == list(wv.NAMES) and d["decompositions"]["wavelet-LLL"]["bin_width"] == 50
    assert d["decompositions"]["wavelet-LLH"]["firstorder"] == json.loads(json.dumps(f["LLH"].first_order.to_dict()))
    assert d["decompositions"]["wavelet-LLH"]["texture"] == json.loads(json.dumps(f["LLH"].texture.to_dict()))
    save_wavelet_features(str(tmp_path / "w.csv"), f)
    with open(tmp_path / "w.csv") as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["label", "name", "voxels"] + list(f.vector(1))
    assert [r[:3] for r in rows[1:]] == [["1", "left", "64"], ["lung", "lung", "64"]]
    for r, label in zip(rows[1:], (1, "lung")):
        want = f.vector(label)
        for k, cell in zip(rows[0][3:], r[3:]):
            assert float(cell) == want[k] or (math.isnan(float(cell)) and math.isnan(want[k])), k
    with pytest.raises(SystemExit):
        save_wavelet_features(str(tmp_path / "w.txt"), f)


def test_cli_flags_and_checks_before_segmentation(tmp_path):
    from lungmask_b200.__main__ import build_parser, main
    inp = tmp_path / "in.npy"
    np.save(inp, np.zeros((2, 8, 8), np.int16))
    a = build_parser().parse_args([str(inp), "out.npy"])
    assert (a.wavelet, a.wavelet_name, a.wavelet_bin_width) == (None, "coif1", "25")
    assert a.wavelet_classes == "firstorder,glcm,glszm,glrlm,gldm,ngtdm"
    a = build_parser().parse_args([str(inp), "out.npy", "--wavelet", "w.csv", "--wavelet-name", "haar",
                                   "--wavelet-bin-width", "25,LLL=50", "--wavelet-classes", "firstorder,glcm"])
    assert (a.wavelet, a.wavelet_name, a.wavelet_bin_width, a.wavelet_classes) == ("w.csv", "haar", "25,LLL=50",
                                                                                  "firstorder,glcm")
    with pytest.raises(SystemExit):
        build_parser().parse_args([str(inp), "out.npy", "--wavelet-name", "db2"])
    out = str(tmp_path / "m.npy")
    # every check ends the run before the volume is segmented (that would need a model and a GPU)
    for extra, msg in (((), "unsupported wavelet output"),
                       (("--wavelet-bin-width", "0"), "wavelet-bin-width"),
                       (("--wavelet-bin-width", "25,XYZ=3"), "wavelet-bin-width"),
                       (("--wavelet-classes", "glcm,shape"), "wavelet-classes")):
        path = str(tmp_path / ("w.xlsx" if not extra else "w.json"))
        with pytest.raises(SystemExit, match=msg):
            main([str(inp), out, "--wavelet", path, *extra])
