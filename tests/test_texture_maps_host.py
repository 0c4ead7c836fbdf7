"""The numpy statement of the voxel-based GLSZM, GLRLM, GLDM and NGTDM maps (texture_maps.maps_host) against a literal
per-voxel loop over texture's feature functions, exact Fractions, the integer bounds at worst-case windows, and the
argument checks, writer and CLI checks (CPU only)."""
import math
from fractions import Fraction

import numpy as np
import pytest
from scipy import ndimage

from lungmask_b200 import first_order_maps as fm
from lungmask_b200 import glcm_maps as gm
from lungmask_b200 import texture as tx
from lungmask_b200 import texture_maps as tm

CUBE = np.ones((3, 3, 3), bool)
NEIGH = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1) if a or b or c]


def window_of(lev, c, r):
    """The window of centre c: the levels of the (2r+1)^3 cube about c, clipped at the array border."""
    sl = tuple(slice(max(c[k] - r, 0), c[k] + r + 1) for k in range(3))
    return lev[sl]


def literal_window(win, ng, alpha):
    """The four classes' features of one window (levels, 0 = not a candidate), each matrix built on its own."""
    n_p = int((win > 0).sum())
    zl, zs, zc = [], [], []
    for level in range(1, ng + 1):
        lab, k = ndimage.label(win == level, structure=CUBE)
        if k:
            sizes, counts = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
            zl += [level] * len(sizes)
            zs += list(sizes)
            zc += list(counts)
    glszm = tx.glszm_features(zl, zs, zc, n_p)
    E = max(win.shape)
    runs = np.zeros((13, ng, E), np.int64)
    G = np.zeros((ng, 27), np.int64)
    N = np.zeros((ng, 27), np.int64)
    A = np.zeros((ng, 27), np.int64)
    inside = lambda q: all(0 <= q[k] < win.shape[k] for k in range(3))   # noqa: E731
    for p in zip(*np.nonzero(win)):
        i = int(win[p])
        for d, off in enumerate(tx.OFFSETS):
            b = tuple(p[k] - off[k] for k in range(3))
            if inside(b) and win[b] == i:
                continue
            n, q = 1, tuple(p[k] + off[k] for k in range(3))
            while inside(q) and win[q] == i:
                n += 1
                q = tuple(q[k] + off[k] for k in range(3))
            runs[d, i - 1, n - 1] += 1
        w = s = dep = 0
        for off in NEIGH:
            q = tuple(p[k] + off[k] for k in range(3))
            if inside(q) and win[q]:
                w += 1
                s += int(win[q])
                dep += abs(int(win[q]) - i) <= alpha
        G[i - 1, dep] += 1
        N[i - 1, w] += 1
        A[i - 1, w] += abs(w * i - s)
    return {"glszm": glszm, "glrlm": tx.glrlm_features(runs), "gldm": tx.gldm_features(G),
            "ngtdm": tx.ngtdm_features(N, A)}


def literal_maps(vol, mask, label, r, masked, bw, alpha=0):
    roi = fm.roi_of(vol, mask, label)
    lev, low, ng = gm.level_map(vol, fm.region(vol, roi, r, masked), bw)
    return {c: literal_window(window_of(lev, c, r), ng, alpha) for c in zip(*np.nonzero(roi))}


def assert_maps_match(res, lit):
    for c, per in lit.items():
        for cls in res.classes:
            for k, want in per[cls].items():
                got = res.maps["%s_%s" % (cls, k)][c]
                if math.isnan(want):
                    assert math.isnan(got), (c, cls, k, got)
                else:
                    assert abs(got - want) <= 1e-12 * max(abs(want), 1.0), (c, cls, k, got, want)


def volume(kind, shape, rng):
    if kind == "int16":
        return rng.integers(-1000, -700, shape).astype(np.int16)
    if kind == "int32":
        return rng.integers(-(1 << 20), 1 << 20, shape).astype(np.int32)
    v = (rng.normal(-800, 80, shape)).astype(np.float32)
    v[rng.random(shape) < 0.1] = np.nan
    return v


@pytest.mark.parametrize("kind", ["int16", "int32", "float32"])
@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("masked", [True, False])
def test_maps_host_against_loop(kind, r, masked):
    rng = np.random.default_rng(7 * r + (kind == "float32") + 3 * masked)
    shape = (4, 5, 6)
    vol = volume(kind, shape, rng)
    mask = rng.integers(0, 3, shape).astype(np.uint8)
    bw = 25 if kind != "int32" else 1 << 17
    res = tm.maps_host(vol, mask, "lung", kernel_radius=r, masked_kernel=masked, bin_width=bw)
    assert_maps_match(res, literal_maps(vol, mask, "lung", r, masked, bw))


@pytest.mark.parametrize("alpha", [0, 2])
def test_gldm_alpha_against_loop(alpha):
    rng = np.random.default_rng(3 + alpha)
    vol = rng.integers(-1000, -850, (5, 6, 6)).astype(np.int16)
    mask = rng.integers(0, 2, vol.shape).astype(np.uint8)
    res = tm.maps_host(vol, mask, classes=("gldm",), kernel_radius=2, gldm_alpha=alpha, bin_width=25)
    assert res.gldm_alpha == alpha and list(res.maps) == ["gldm_" + f for f in tx.GLDM_FEATURES]
    assert_maps_match(res, literal_maps(vol, mask, "lung", 2, True, 25, alpha))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 2, 1), (2, 1, 2), (1, 4, 3), (3, 1, 1)])
@pytest.mark.parametrize("init", [0.0, float("nan")])
def test_small_extents_label_row_and_init_value(shape, init):
    rng = np.random.default_rng(11)
    vol = rng.integers(-1000, -800, shape).astype(np.int16)
    mask = rng.integers(0, 3, shape).astype(np.uint8)
    mask.reshape(-1)[0] = 2
    res = tm.maps_host(vol, mask, 2, kernel_radius=2, init_value=init)
    assert_maps_match(res, literal_maps(vol, mask, 2, 2, True, 25))
    outside = mask != 2
    for k, m in res.maps.items():
        assert m.shape == shape and m.dtype == np.float64
        assert np.isnan(m[outside]).all() if math.isnan(init) else (m[outside] == init).all()


def test_isolated_centres():
    """A speckle ROI: one-voxel zones and runs, dependence size 1, and NGTDM NaN (no voxel has a neighbour)."""
    vol = np.arange(5 * 6 * 7, dtype=np.int16).reshape(5, 6, 7) - 900
    mask = np.zeros(vol.shape, np.uint8)
    mask[::2, ::2, ::2] = 1
    res = tm.maps_host(vol, mask, kernel_radius=1, init_value=-2.0)
    on = mask == 1
    for k in tx.NGTDM_FEATURES:
        assert np.isnan(res["ngtdm_" + k][on]).all() and (res["ngtdm_" + k][~on] == -2.0).all(), k
    assert (res["glszm_SmallAreaEmphasis"][on] == 1.0).all() and (res["glszm_ZonePercentage"][on] == 1.0).all()
    assert (res["glrlm_ShortRunEmphasis"][on] == 1.0).all()
    assert (res["gldm_SmallDependenceEmphasis"][on] == 1.0).all()
    assert not np.isnan(tm.maps_host(vol, mask, masked_kernel=False)["ngtdm_Contrast"][on]).any()


@pytest.mark.parametrize("r", [1, 2, 3])
def test_cover_case_equals_row_features(r):
    """A ROI inside an (r+1)^3 cube: every window holds the whole ROI, so every map equals the row's features."""
    rng = np.random.default_rng(60 + r)
    vol = rng.integers(-1000, -800, (8, 9, 10)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    e = r + 1
    mask[2:2 + e, 3:3 + e, 3:3 + e] = rng.integers(0, 2, (e, e, e)).astype(np.uint8) * 3
    mask[2, 3, 3] = 3
    res = tm.maps_host(vol, mask, 3, kernel_radius=r)
    lev, _, ng = gm.level_map(vol, mask == 3, 25)
    row = literal_window(lev, ng, 0)
    for cls in tm.CLASSES:
        for k, want in row[cls].items():
            got = res["%s_%s" % (cls, k)][mask == 3]
            assert np.allclose(got, want, rtol=1e-12, atol=1e-12), (cls, k)


def _ulps(got, exact):
    want = float(exact)
    if got == want:
        return 0.0
    return float(abs(Fraction(got) - exact) / Fraction(np.spacing(abs(want)) if want else np.spacing(0.0)))


def _fraction_zone_features(entries, n_p):
    """The exact rational GLSZM features of (i, s, c) entries."""
    nz = sum(c for _, _, c in entries)
    p = [(i, s, Fraction(c, nz)) for i, s, c in entries]
    gi, gs = {}, {}
    for i, s, c in entries:
        gi[i] = gi.get(i, 0) + c
        gs[s] = gs.get(s, 0) + c
    mi = sum(q * i for i, s, q in p)
    ms = sum(q * s for i, s, q in p)
    return {"LargeAreaEmphasis": sum(q * s * s for i, s, q in p),
            "GrayLevelNonUniformity": Fraction(sum(v * v for v in gi.values()), nz),
            "GrayLevelNonUniformityNormalized": Fraction(sum(v * v for v in gi.values()), nz * nz),
            "SizeZoneNonUniformity": Fraction(sum(v * v for v in gs.values()), nz),
            "SizeZoneNonUniformityNormalized": Fraction(sum(v * v for v in gs.values()), nz * nz),
            "ZonePercentage": Fraction(nz, n_p), "GrayLevelVariance": sum(q * (i - mi) ** 2 for i, s, q in p),
            "ZoneVariance": sum(q * (s - ms) ** 2 for i, s, q in p),
            "HighGrayLevelZoneEmphasis": sum(q * i * i for i, s, q in p),
            "LargeAreaHighGrayLevelEmphasis": sum(q * i * i * s * s for i, s, q in p)}


@pytest.mark.parametrize("r", [1, 2, 3])
def test_rational_glszm_features_within_two_ulp(r):
    rng = np.random.default_rng(40 + r)
    vol = rng.integers(-1000, -700, (6, 7, 8)).astype(np.int16)
    mask = rng.integers(0, 2, vol.shape).astype(np.uint8)
    res = tm.maps_host(vol, mask, classes=("glszm",), kernel_radius=r, bin_width=25)
    lev, _, ng = gm.level_map(vol, mask > 0, 25)
    for c in list(zip(*np.nonzero(mask)))[::5]:
        win = window_of(lev, c, r)
        ent = {}
        for level in range(1, ng + 1):
            lab, k = ndimage.label(win == level, structure=CUBE)
            for s in np.bincount(lab.ravel())[1:]:
                ent[(level, int(s))] = ent.get((level, int(s)), 0) + 1
        exact = _fraction_zone_features([(i, s, n) for (i, s), n in sorted(ent.items())], int((win > 0).sum()))
        for k, v in exact.items():
            assert _ulps(res["glszm_" + k][c], v) <= 2.0, (c, k, res["glszm_" + k][c], float(v))


def test_rational_ngtdm_features_within_two_ulp():
    rng = np.random.default_rng(9)
    vol = rng.integers(-1000, -600, (5, 6, 7)).astype(np.int16)
    mask = rng.integers(0, 2, vol.shape).astype(np.uint8)
    res = tm.maps_host(vol, mask, classes=("ngtdm",), kernel_radius=2, bin_width=25)
    lev, _, ng = gm.level_map(vol, mask > 0, 25)
    for c in list(zip(*np.nonzero(mask)))[::3]:
        win = window_of(lev, c, 2)
        n, s = {}, {}
        for p in zip(*np.nonzero(win)):
            w = t = 0
            for off in NEIGH:
                q = tuple(p[k] + off[k] for k in range(3))
                if all(0 <= q[k] < win.shape[k] for k in range(3)) and win[q]:
                    w, t = w + 1, t + int(win[q])
            if w:
                i = int(win[p])
                n[i] = n.get(i, 0) + 1
                s[i] = s.get(i, 0) + abs(Fraction(w * i - t, w))
        if not n:
            continue
        nvp = sum(n.values())
        ps = sum(Fraction(n[i], nvp) * s[i] for i in n)
        busy = sum(abs(Fraction(i * n[i] - j * n[j], nvp)) for i in n for j in n)
        ss = sum(s.values())
        exact = {"Coarseness": 1 / ps if ps else None, "Busyness": ps / busy if busy else Fraction(0),
                 "Strength": sum(Fraction(n[i] + n[j], nvp) * (i - j) ** 2 for i in n for j in n) / ss if ss else Fraction(0)}
        for k, v in exact.items():
            if v is not None:
                assert _ulps(res["ngtdm_" + k][c], v) <= 2.0, (c, k)


def test_integer_bounds_at_worst_case_windows():
    """A uniform 343-voxel window (one zone, runs of 7, dependence size 27) and a checkerboard at Ng = 255: the integer
    sums stay exact and the features equal their closed forms."""
    vol = np.full((7, 7, 7), 254 * 25, np.int16)
    vol[0, 0, 0] = 0   # Ng = 255; the level-255 zone holds 342 voxels around the one level-1 voxel
    mask = np.ones(vol.shape, np.uint8)
    res = tm.maps_host(vol, mask, classes=("glszm", "glrlm", "gldm"), kernel_radius=3, bin_width=25,
                       features=("glszm_LargeAreaHighGrayLevelEmphasis", "glszm_ZonePercentage",
                                 "glrlm_LongRunHighGrayLevelEmphasis", "gldm_LargeDependenceHighGrayLevelEmphasis"))
    c = (3, 3, 3)
    assert res.n_levels == 255
    assert res["glszm_LargeAreaHighGrayLevelEmphasis"][c] == float(Fraction(255 ** 2 * 342 ** 2 + 1, 2))
    assert res["glszm_ZonePercentage"][c] == 2 / 343
    uni = np.full((7, 7, 7), -900, np.int16)
    res = tm.maps_host(uni, mask, kernel_radius=3, bin_width=25)
    assert res["glszm_LargeAreaEmphasis"][c] == 343.0 ** 2 and res["glszm_ZonePercentage"][c] == 1 / 343
    # dependence sizes in a full 7^3 window: 8 corners 8, 60 edge voxels 12, 150 face voxels 18, 125 inner voxels 27
    assert res["gldm_LargeDependenceEmphasis"][c] == float(Fraction(8 * 8 ** 2 + 60 * 12 ** 2 + 150 * 18 ** 2 +
                                                                    125 * 27 ** 2, 343))
    assert res["ngtdm_Coarseness"][c] == 1e6 and res["ngtdm_Busyness"][c] == 0.0 and res["ngtdm_Strength"][c] == 0.0
    # checkerboard of levels 1 and 255: every voxel's neighbours are mixed, sigma_i near its 343 * 254 L bound
    z, y, x = np.indices((7, 7, 7))
    chk = np.where((z + y + x) % 2 == 0, 0, 254 * 25).astype(np.int16)
    res = tm.maps_host(chk, mask, kernel_radius=3, bin_width=25)
    lit = literal_window(gm.level_map(chk, mask > 0, 25)[0], 255, 0)
    assert res.n_levels == 255
    for cls in tm.CLASSES:
        for k, want in lit[cls].items():
            assert abs(res["%s_%s" % (cls, k)][c] - want) <= 1e-12 * max(abs(want), 1.0), (cls, k)


def test_refusals():
    vol = np.random.default_rng(1).normal(-800, 50, (4, 6, 6)).astype(np.float32)
    mask = np.ones(vol.shape, np.uint8)
    with pytest.raises(ValueError, match="kernel_radius"):
        tm.maps_host(vol, mask, kernel_radius=0)
    with pytest.raises(ValueError, match="label"):
        tm.maps_host(vol, mask, label=256)
    with pytest.raises(ValueError, match="glcm_maps"):
        tm.maps_host(vol, mask, classes=("glcm", "glszm"))
    with pytest.raises(ValueError, match="unknown texture class"):
        tm.check_classes(("glszm", "lbp"))
    with pytest.raises(TypeError):
        tm.check_classes("glszm")
    with pytest.raises(ValueError, match="at least one"):
        tm.check_classes(())
    with pytest.raises(ValueError, match="unknown feature"):
        tm.maps_host(vol, mask, features=("glszm_ZoneEntropy", "glszm_Bogus"))
    with pytest.raises(ValueError, match="unknown feature"):
        tm.check_features(("ZoneEntropy",), tm.CLASSES)
    with pytest.raises(ValueError, match="not among the requested"):
        tm.maps_host(vol, mask, classes=("glszm",), features=("ngtdm_Contrast",))
    with pytest.raises(TypeError):
        tm.check_features("glszm_ZoneEntropy", tm.CLASSES)
    with pytest.raises(ValueError, match="empty"):
        tm.check_features((), tm.CLASSES)
    with pytest.raises(ValueError, match="gldm_alpha"):
        tm.maps_host(vol, mask, gldm_alpha=-1)
    with pytest.raises(TypeError, match="gldm_alpha"):
        tm.maps_host(vol, mask, gldm_alpha=1.5)
    with pytest.raises(ValueError, match="bin_width"):
        tm.maps_host(vol, mask, bin_width=0)
    with pytest.raises(ValueError, match="grey levels"):
        tm.maps_host(vol * 100, mask, bin_width=1)
    bad = vol.copy()
    bad[1, 2, 2] = -np.inf
    with pytest.raises(ValueError, match="non-finite"):
        tm.maps_host(bad, mask)
    assert tm.check_features(("ngtdm_Contrast", "glszm_ZoneEntropy"), tm.CLASSES) == ("glszm_ZoneEntropy", "ngtdm_Contrast")
    assert len(tm.check_features(None, tm.CLASSES)) == 51
    feats = tm.check_features(None, tm.CLASSES)
    assert [tm.feature_bits(feats, c) for c in tm.CLASSES] == [(1 << 16) - 1, (1 << 16) - 1, (1 << 14) - 1, (1 << 5) - 1]
    assert tm.feature_bits(("ngtdm_Busyness",), "ngtdm") == 4 and tm.feature_bits(("ngtdm_Busyness",), "glszm") == 0


def test_writer_names_and_round_trip(tmp_path):
    from lungmask_b200.io import load_input_image, save_feature_maps
    vol = np.random.default_rng(2).integers(-1000, -700, (3, 8, 9)).astype(np.int16)
    mask = np.ones(vol.shape, np.uint8)
    res = tm.maps_host(vol, mask, 1, features=("glszm_SmallAreaEmphasis", "ngtdm_Contrast"), init_value=float("nan"))
    paths = save_feature_maps(str(tmp_path), res, None, "nii.gz")
    assert sorted(p.split("/")[-1] for p in paths) == ["1_glszm_SmallAreaEmphasis.nii.gz", "1_ngtdm_Contrast.nii.gz"]
    for k in ("glszm_SmallAreaEmphasis", "ngtdm_Contrast"):
        img = load_input_image(str(tmp_path / ("1_%s.nii.gz" % k)))
        assert np.array_equal(np.asarray(img.array).view(np.uint64), res[k].view(np.uint64))


@pytest.mark.parametrize("argv, msg", [
    (["--texture-maps-label", "0"], "--texture-maps-label"),
    (["--texture-maps-label", "x"], None),
    (["--texture-maps-features", "glszm_ZoneEntropy,Bogus"], "--texture-maps-features"),
    (["--texture-maps-classes", "glszm,glcm"], "--texture-maps-classes"),
    (["--texture-maps-classes", "glszm", "--texture-maps-features", "ngtdm_Contrast"], "--texture-maps-features"),
    (["--texture-bin-width", "0"], "--texture-bin-width"),
])
def test_cli_argument_checks(tmp_path, argv, msg):
    from lungmask_b200.__main__ import build_parser, texture_maps_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    args = build_parser().parse_args([str(src), "out.nii", "--texture-maps", str(tmp_path / "maps")] + argv)
    with pytest.raises((SystemExit, ValueError)) as e:
        texture_maps_arguments(args)
    if msg is not None:
        assert msg in str(e.value)


def test_cli_checks_the_directory_and_defaults(tmp_path):
    from lungmask_b200.__main__ import build_parser, texture_maps_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    f = tmp_path / "file"
    f.write_text("x")
    args = build_parser().parse_args([str(src), "out.nii", "--texture-maps", str(f)])
    with pytest.raises(SystemExit, match="not a directory"):
        texture_maps_arguments(args)
    args = build_parser().parse_args([str(src), "out.nii", "--texture-maps", str(tmp_path / "a" / "b")])
    with pytest.raises(SystemExit, match="parent directory"):
        texture_maps_arguments(args)
    args = build_parser().parse_args([str(src), "out.nii", "--texture-maps", str(tmp_path / "m"), "--texture-maps-label",
                                      "3", "--texture-maps-classes", "ngtdm, glszm", "--texture-maps-features",
                                      "ngtdm_Contrast, glszm_ZoneEntropy", "--texture-maps-radius", "3",
                                      "--texture-maps-unmasked"])
    assert texture_maps_arguments(args) == (3, ("glszm", "ngtdm"), ("glszm_ZoneEntropy", "ngtdm_Contrast"))
    assert args.texture_maps_radius == 3 and args.texture_maps_unmasked and args.texture_maps_format == "nii.gz"
    args = build_parser().parse_args([str(src), "out.nii", "--texture-maps", str(tmp_path / "m")])
    assert texture_maps_arguments(args) == ("lung", tm.CLASSES, None)
    with pytest.raises(SystemExit):
        build_parser().parse_args([str(src), "out.nii", "--texture-maps", "d", "--texture-maps-radius", "4"])
