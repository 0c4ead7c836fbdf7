"""The numpy statement of the voxel-based GLCM maps (glcm_maps.maps_host) against a literal per-voxel loop over
texture.glcm_features, exact Fractions and mpmath, and the argument checks, writer and CLI checks (CPU only)."""
import math
from fractions import Fraction

import numpy as np
import pytest

from lungmask_b200 import first_order_maps as fm
from lungmask_b200 import glcm_maps as gm
from lungmask_b200 import texture as tx

RATIONAL = ("Autocorrelation", "JointAverage", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast",
            "Correlation", "DifferenceAverage", "DifferenceVariance", "JointEnergy", "MaximumProbability", "SumSquares")


def window_counts(lev, c, r):
    """U (13, ng (ng + 1) / 2) of the window of c over a level map (0 = not a candidate), counted pair by pair."""
    ng = int(lev.max())
    iu = {(i, j): k for k, (i, j) in enumerate(zip(*np.triu_indices(ng)))}
    U = np.zeros((13, len(iu)), np.int64)
    S, H, W = lev.shape
    inside = lambda p: all(abs(p[k] - c[k]) <= r for k in range(3)) and 0 <= p[0] < S and 0 <= p[1] < H and 0 <= p[2] < W
    for d, off in enumerate(tx.OFFSETS):
        for z in range(max(c[0] - r, 0), min(c[0] + r + 1, S)):
            for y in range(max(c[1] - r, 0), min(c[1] + r + 1, H)):
                for x in range(max(c[2] - r, 0), min(c[2] + r + 1, W)):
                    q = (z + off[0], y + off[1], x + off[2])
                    if inside(q) and lev[z, y, x] and lev[q]:
                        a, b = sorted((int(lev[z, y, x]), int(lev[q])))
                        U[d, iu[(a - 1, b - 1)]] += 1
    return U


def literal_maps(vol, mask, label, r, masked, bw):
    """Per ROI voxel: its window's pair counts through texture.glcm_features, in a plain loop."""
    roi = fm.roi_of(vol, mask, label)
    lev, low, ng = gm.level_map(vol, fm.region(vol, roi, r, masked), bw)
    return {c: (window_counts(lev, c, r), tx.glcm_features(window_counts(lev, c, r), ng)) for c in zip(*np.nonzero(roi))}


def assert_maps_match(res, lit):
    for c, (_, f) in lit.items():
        for k in gm.FEATURES:
            got, want = res.maps[k][c], f[k]
            if math.isnan(want):
                assert math.isnan(got), (c, k, got)
            elif k == "Imc2":
                # sqrt(1 - exp(-2 d)) with d = HXY2 - HXY: |d| errors of both sides reach the square, not the root
                assert abs(got * got - want * want) <= 1e-12 * max(1.0, want * want), (c, k, got, want)
            else:
                assert abs(got - want) <= 1e-12 * max(abs(want), 1.0), (c, k, got, want)


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
    bw = 25 if kind != "int32" else 1 << 14
    res = gm.maps_host(vol, mask, "lung", kernel_radius=r, masked_kernel=masked, bin_width=bw)
    assert_maps_match(res, literal_maps(vol, mask, "lung", r, masked, bw))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 2, 1), (2, 1, 2), (1, 4, 3), (3, 1, 1)])
@pytest.mark.parametrize("init", [0.0, float("nan")])
def test_small_extents_label_row_and_init_value(shape, init):
    rng = np.random.default_rng(11)
    vol = rng.integers(-1000, -800, shape).astype(np.int16)
    mask = rng.integers(0, 3, shape).astype(np.uint8)
    mask.reshape(-1)[0] = 2
    res = gm.maps_host(vol, mask, 2, kernel_radius=2, init_value=init)
    assert_maps_match(res, literal_maps(vol, mask, 2, 2, True, 25))
    outside = mask != 2
    for k, m in res.maps.items():
        assert m.shape == shape and m.dtype == np.float64
        assert np.isnan(m[outside]).all() if math.isnan(init) else (m[outside] == init).all()


def test_isolated_roi_voxels_are_nan():
    vol = np.arange(5 * 6 * 7, dtype=np.int16).reshape(5, 6, 7) - 900
    mask = np.zeros(vol.shape, np.uint8)
    mask[::2, ::2, ::2] = 1
    res = gm.maps_host(vol, mask, kernel_radius=1, init_value=-2.0)
    for k in gm.FEATURES:
        assert np.isnan(res[k][mask == 1]).all(), k
        assert (res[k][mask == 0] == -2.0).all(), k
    # unmasked, the same voxels see their neighbours
    assert not np.isnan(gm.maps_host(vol, mask, kernel_radius=1, masked_kernel=False)["Contrast"][mask == 1]).any()


def _fraction_features(U, ng):
    """The exact rational features of one direction's pair counts."""
    P = {}
    iu, ju = np.triu_indices(ng)
    for u, i, j in zip(U, iu + 1, ju + 1):
        if u:
            P[(i, j)] = P.get((i, j), 0) + int(u)
            P[(j, i)] = P.get((j, i), 0) + int(u)
    N = sum(P.values())
    p = {k: Fraction(v, N) for k, v in P.items()}
    mu = sum(i * q for (i, j), q in p.items())
    sx2 = sum((i - mu) ** 2 * q for (i, j), q in p.items())
    da = sum(abs(i - j) * q for (i, j), q in p.items())
    f = {"Autocorrelation": sum(i * j * q for (i, j), q in p.items()), "JointAverage": mu,
         "ClusterProminence": sum((i + j - 2 * mu) ** 4 * q for (i, j), q in p.items()),
         "ClusterShade": sum((i + j - 2 * mu) ** 3 * q for (i, j), q in p.items()),
         "ClusterTendency": sum((i + j - 2 * mu) ** 2 * q for (i, j), q in p.items()),
         "Contrast": sum((i - j) ** 2 * q for (i, j), q in p.items()),
         "Correlation": Fraction(1) if sx2 == 0 else sum((i - mu) * (j - mu) * q for (i, j), q in p.items()) / sx2,
         "DifferenceAverage": da,
         "DifferenceVariance": sum((abs(i - j) - da) ** 2 * q for (i, j), q in p.items()),
         "JointEnergy": sum(q * q for q in p.values()), "MaximumProbability": max(p.values()), "SumSquares": sx2}
    return f


def _ulps(got, exact):
    want = float(exact)
    if got == want:
        return 0.0
    return float(abs(Fraction(got) - exact) / Fraction(np.spacing(abs(want)) if want else np.spacing(0.0)))


@pytest.mark.parametrize("r", [1, 2, 3])
def test_rational_features_within_two_ulp(r):
    """Lines along one axis: each window has pairs in one direction only, so its map value is that direction's."""
    rng = np.random.default_rng(40 + r)
    for shape in ((1, 1, 41), (1, 33, 1), (29, 1, 1)):
        vol = rng.integers(-1000, 2000, shape).astype(np.int16)
        mask = np.ones(shape, np.uint8)
        res = gm.maps_host(vol, mask, kernel_radius=r, bin_width=25)
        lev, _, ng = gm.level_map(vol, mask > 0, 25)
        for c in zip(*np.nonzero(mask)):
            U = window_counts(lev, c, r)
            d = int(np.nonzero(U.any(axis=1))[0][0])
            exact = _fraction_features(U[d], ng)
            for k in RATIONAL:
                assert _ulps(res[k][c], exact[k]) <= 2.0, (shape, c, k, res[k][c], float(exact[k]))


@pytest.mark.parametrize("r", [1, 2, 3])
def test_cover_case_equals_row_features(r):
    """A ROI inside an (r+1)^3 cube: every window holds the whole ROI, so every map equals the row's GLCM features."""
    rng = np.random.default_rng(60 + r)
    vol = rng.integers(-1000, -400, (8, 9, 10)).astype(np.int16)
    mask = np.zeros(vol.shape, np.uint8)
    e = r + 1
    mask[2:2 + e, 3:3 + e, 3:3 + e] = rng.integers(0, 2, (e, e, e)).astype(np.uint8) * 3
    mask[2, 3, 3] = 3
    res = gm.maps_host(vol, mask, 3, kernel_radius=r)
    lev, _, ng = gm.level_map(vol, mask == 3, 25)
    U = np.zeros((13, ng * (ng + 1) // 2), np.int64)
    iu = {(i, j): k for k, (i, j) in enumerate(zip(*np.triu_indices(ng)))}
    for d, off in enumerate(tx.OFFSETS):
        for p in zip(*np.nonzero(lev)):
            q = tuple(p[k] + off[k] for k in range(3))
            if all(0 <= q[k] < lev.shape[k] for k in range(3)) and lev[q]:
                a, b = sorted((int(lev[p]), int(lev[q])))
                U[d, iu[(a - 1, b - 1)]] += 1
    row = tx.glcm_features(U, ng)
    for k in gm.FEATURES:
        got = res[k][mask == 3]
        assert np.allclose(got, row[k], rtol=1e-12, atol=1e-12), k


def test_log2_and_exp_routines_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.dps = 50
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.random(3000), np.exp(rng.uniform(-700, 700, 3000)), 1 + rng.uniform(-1e-6, 1e-6, 500),
                        [1.0, 2.0 ** -52, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, np.nextafter(1, 0),
                         np.nextafter(1, 2), math.sqrt(2), np.nextafter(math.sqrt(2), 3), 0.5, 3.0, 1 + 2.0 ** -52]])
    got = gm.log2_fixed(x)
    for xi, g in zip(x, got):
        ex = mpmath.log(mpmath.mpf(float(xi)), 2)
        if ex == 0:
            assert g == 0.0
            continue
        assert abs(mpmath.mpf(float(g)) - ex) <= gm.LOG2_ULP * mpmath.mpf(float(np.spacing(abs(float(ex))))), xi
    lo, hi = gm.EXP_DOMAIN
    y = np.concatenate([rng.uniform(lo, hi, 3000), rng.uniform(-1, 1, 2000), rng.uniform(-1e-8, 1e-8, 300),
                        [0.0, -0.0, lo, hi, 0.34657359027997264, -0.34657359027997264, -40.0, 1e-300, -1e-300]])
    got = gm.exp_fixed(y)
    for yi, g in zip(y, got):
        ex = mpmath.exp(mpmath.mpf(float(yi)))
        assert abs(mpmath.mpf(float(g)) - ex) <= gm.EXP_ULP * mpmath.mpf(float(np.spacing(float(ex)))), yi
    assert (gm.exp_fixed(-np.linspace(0, 40, 1001)) <= 1.0).all()   # Imc2's 1 - exp(y) never goes negative


def test_refusals():
    vol = np.random.default_rng(1).normal(-800, 50, (4, 6, 6)).astype(np.float32)
    mask = np.ones(vol.shape, np.uint8)
    with pytest.raises(ValueError, match="kernel_radius"):
        gm.maps_host(vol, mask, kernel_radius=0)
    with pytest.raises(ValueError, match="label"):
        gm.maps_host(vol, mask, label=256)
    with pytest.raises(ValueError, match="unknown GLCM feature"):
        gm.maps_host(vol, mask, features=("Contrast", "MCC"))
    with pytest.raises(TypeError):
        gm.check_features("Contrast")
    with pytest.raises(ValueError, match="empty"):
        gm.check_features(())
    with pytest.raises(ValueError, match="bin_width"):
        gm.maps_host(vol, mask, bin_width=0)
    with pytest.raises(ValueError, match="grey levels"):
        gm.maps_host(vol * 100, mask, bin_width=1)
    bad = vol.copy()
    bad[1, 2, 2] = -np.inf
    with pytest.raises(ValueError, match="non-finite"):
        gm.maps_host(bad, mask)
    assert gm.check_features(("Idm", "Contrast")) == ("Contrast", "Idm")
    assert gm.feature_bits(gm.FEATURES) == (1 << 22) - 1


def test_writer_names_and_round_trip(tmp_path):
    from lungmask_b200.io import feature_map_file, load_input_image, save_feature_maps
    assert feature_map_file("lung", "Contrast", "nii.gz", "glcm") == "lung_glcm_Contrast.nii.gz"
    assert feature_map_file("lung", "Entropy", "nii.gz") == "lung_Entropy.nii.gz"
    vol = np.random.default_rng(2).integers(-1000, -700, (3, 8, 9)).astype(np.int16)
    mask = np.ones(vol.shape, np.uint8)
    res = gm.maps_host(vol, mask, 1, features=("JointEntropy", "Imc1"), init_value=float("nan"))
    paths = save_feature_maps(str(tmp_path), res, None, "nii.gz")
    assert sorted(p.split("/")[-1] for p in paths) == ["1_glcm_Imc1.nii.gz", "1_glcm_JointEntropy.nii.gz"]
    for k in ("JointEntropy", "Imc1"):
        img = load_input_image(str(tmp_path / ("1_glcm_%s.nii.gz" % k)))
        assert np.array_equal(np.asarray(img.array).view(np.uint64), res[k].view(np.uint64))
    npy = save_feature_maps(str(tmp_path / "n"), res, None, "npy")
    assert np.array_equal(np.load(npy[0]).view(np.uint64), res["JointEntropy"].view(np.uint64))


@pytest.mark.parametrize("argv, msg", [
    (["--glcm-maps-label", "0"], "--glcm-maps-label"),
    (["--glcm-maps-label", "x"], None),
    (["--glcm-maps-features", "Contrast,Bogus"], "--glcm-maps-features"),
    (["--texture-bin-width", "0"], "--texture-bin-width"),
])
def test_cli_argument_checks(tmp_path, argv, msg):
    from lungmask_b200.__main__ import build_parser, glcm_maps_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    args = build_parser().parse_args([str(src), "out.nii", "--glcm-maps", str(tmp_path / "maps")] + argv)
    with pytest.raises((SystemExit, ValueError)) as e:
        glcm_maps_arguments(args)
    if msg is not None:
        assert msg in str(e.value)


def test_cli_checks_the_directory_and_defaults(tmp_path):
    from lungmask_b200.__main__ import build_parser, glcm_maps_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    f = tmp_path / "file"
    f.write_text("x")
    args = build_parser().parse_args([str(src), "out.nii", "--glcm-maps", str(f)])
    with pytest.raises(SystemExit, match="not a directory"):
        glcm_maps_arguments(args)
    args = build_parser().parse_args([str(src), "out.nii", "--glcm-maps", str(tmp_path / "a" / "b")])
    with pytest.raises(SystemExit, match="parent directory"):
        glcm_maps_arguments(args)
    args = build_parser().parse_args([str(src), "out.nii", "--glcm-maps", str(tmp_path / "m"), "--glcm-maps-label", "3",
                                      "--glcm-maps-features", "Idm, Contrast", "--glcm-maps-radius", "3",
                                      "--glcm-maps-unmasked"])
    assert glcm_maps_arguments(args) == (3, ("Contrast", "Idm"))
    assert args.glcm_maps_radius == 3 and args.glcm_maps_unmasked and args.glcm_maps_format == "nii.gz"
    with pytest.raises(SystemExit):
        build_parser().parse_args([str(src), "out.nii", "--glcm-maps", "d", "--glcm-maps-radius", "4"])
