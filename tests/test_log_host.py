"""The numpy statement of the LoG image type (lungmask_b200.laplacian): the coefficients against a literal restatement,
the vectorised line filter against a scalar per-line loop, independent properties of the filters against the Gaussian
and scipy, the names, the refusals, the bin widths and the command line (no GPU)."""
import math

import numpy as np
import pytest

from lungmask_b200 import laplacian as lg


# ---- coefficients --------------------------------------------------------------------------------------------------

def _literal_coefficients(sd, order):
    """The coefficient rules of DESIGN §4.20 restated step by step."""
    a1s, b1s, a2s, b2s = (1.3530, -0.6724, -1.3563), (1.8151, -3.4327, 5.2318), (-0.3531, 0.6724, 0.3446), \
        (0.0902, 0.6100, -2.2355)
    S1, S2 = math.sin(0.6681 / sd), math.sin(2.0787 / sd)
    C1, C2 = math.cos(0.6681 / sd), math.cos(2.0787 / sd)
    E1, E2 = math.exp(-1.3932 / sd), math.exp(-1.3732 / sd)

    def numer(k):
        a1, b1, a2, b2 = a1s[k], b1s[k], a2s[k], b2s[k]
        n0 = a1 + a2
        n1 = E2 * (b2 * S2 - (a2 + 2 * a1) * C2)
        n1 += E1 * (b1 * S1 - (a1 + 2 * a2) * C1)
        n2 = (a1 + a2) * C2 * C1
        n2 -= b1 * C2 * S1 + b2 * C1 * S2
        n2 *= 2 * E1 * E2
        n2 += a2 * E1 * E1 + a1 * E2 * E2
        n3 = E2 * E1 * E1 * (b2 * S2 - a2 * C2)
        n3 += E1 * E2 * E2 * (b1 * S1 - a1 * C1)
        return [n0, n1, n2, n3], n0 + n1 + n2 + n3, n1 + 2 * n2 + 3 * n3, n1 + 4 * n2 + 9 * n3

    d1 = -2 * E2 * C2 - 2 * E1 * C1
    d2 = 4 * C2 * C1 * E1 * E2 + E1 * E1 + E2 * E2
    d3 = -2 * C1 * E1 * E2 * E2 - 2 * C2 * E2 * E1 * E1
    d4 = E1 * E1 * E2 * E2
    sd_, dd, ed = 1 + d1 + d2 + d3 + d4, d1 + 2 * d2 + 3 * d3 + 4 * d4, d1 + 4 * d2 + 9 * d3 + 16 * d4
    n, sn, dn, en = numer(0)
    if order == 0:
        alpha = 2 * sn / sd_ - n[0]
        n = [x / alpha for x in n]
    else:
        nb, snb, dnb, enb = numer(2)
        beta = -(2 * snb - sd_ * nb[0]) / (2 * sn - sd_ * n[0])
        n = [nb[i] + beta * n[i] for i in range(4)]
        sn, dn, en = snb + beta * sn, dnb + beta * dn, enb + beta * en
        alpha = (en * sd_ * sd_ - ed * sn * sd_ - 2 * dn * dd * sd_ + 2 * dd * dd * sn) / (sd_ * sd_ * sd_)
        n = [x * (sd * sd / alpha) for x in n]
    d = [d1, d2, d3, d4]
    m = [n[1] - d1 * n[0], n[2] - d2 * n[0], n[3] - d3 * n[0], -d4 * n[0]]
    bn = [di * (n[0] + n[1] + n[2] + n[3]) / sd_ for di in d]
    bm = [di * (m[0] + m[1] + m[2] + m[3]) / sd_ for di in d]
    return n + m + d + bn + bm


@pytest.mark.parametrize("sd", [0.25, 0.5, 0.7, 1.0, 1.6, 2.5, 4.0, 5.0 / 0.7, 8.0])
@pytest.mark.parametrize("order", [0, 2])
def test_coefficients_match_literal(sd, order):
    got = lg.coefficients(sd, order).flat()
    want = _literal_coefficients(sd, order)
    assert np.array_equal(np.array(got).view(np.uint64), np.array(want).view(np.uint64))


# ---- the line filter -------------------------------------------------------------------------------------------------

def _scalar_line(x, c):
    """The line filter's rows of DESIGN §4.20, written out per sample for one line of Python floats."""
    x = [float(t) for t in x]
    L, v, w = len(x), x[0], x[-1]
    N0, N1, N2, N3 = c.n
    M1, M2, M3, M4 = c.m
    D1, D2, D3, D4 = c.d
    BN1, BN2, BN3, BN4 = c.bn
    BM1, BM2, BM3, BM4 = c.bm

    def E(a1, b1, a2, b2, a3, b3, a4, b4):
        return ((a1 * b1 + a2 * b2) + a3 * b3) + a4 * b4

    y = [0.0] * L
    y[0] = E(v, N0, v, N1, v, N2, v, N3) - E(v, BN1, v, BN2, v, BN3, v, BN4)
    y[1] = E(x[1], N0, v, N1, v, N2, v, N3) - E(y[0], D1, v, BN2, v, BN3, v, BN4)
    y[2] = E(x[2], N0, x[1], N1, v, N2, v, N3) - E(y[1], D1, y[0], D2, v, BN3, v, BN4)
    y[3] = E(x[3], N0, x[2], N1, x[1], N2, v, N3) - E(y[2], D1, y[1], D2, y[0], D3, v, BN4)
    for i in range(4, L):
        y[i] = E(x[i], N0, x[i - 1], N1, x[i - 2], N2, x[i - 3], N3) - \
            E(y[i - 1], D1, y[i - 2], D2, y[i - 3], D3, y[i - 4], D4)
    z = [0.0] * L
    z[L - 1] = E(w, M1, w, M2, w, M3, w, M4) - E(w, BM1, w, BM2, w, BM3, w, BM4)
    z[L - 2] = E(x[L - 1], M1, w, M2, w, M3, w, M4) - E(z[L - 1], D1, w, BM2, w, BM3, w, BM4)
    z[L - 3] = E(x[L - 2], M1, x[L - 1], M2, w, M3, w, M4) - E(z[L - 2], D1, z[L - 1], D2, w, BM3, w, BM4)
    z[L - 4] = E(x[L - 3], M1, x[L - 2], M2, x[L - 1], M3, w, M4) - E(z[L - 3], D1, z[L - 2], D2, z[L - 1], D3, w, BM4)
    for i in range(L - 4, 0, -1):
        z[i - 1] = E(x[i], M1, x[i + 1], M2, x[i + 2], M3, x[i + 3], M4) - \
            E(z[i], D1, z[i + 1], D2, z[i + 2], D3, z[i + 3], D4)
    return [y[i] + z[i] for i in range(L)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("L", [4, 5, 17, 64])
@pytest.mark.parametrize("sd", [0.25, 0.9, 1.0, 3.3, 8.0])
@pytest.mark.parametrize("order", [0, 2])
def test_line_filter_matches_scalar_loop(L, sd, order):
    rng = np.random.default_rng(L * 100 + int(sd * 10) + order)
    x = rng.normal(0, 300, (L, 6))
    x[:, 0] = -1000.0          # a constant line
    x[:, 1] = np.round(x[:, 1])
    c = lg.coefficients(sd, order)
    got = lg.line_filter(x, c)
    want = np.array([_scalar_line(x[:, k], c) for k in range(x.shape[1])]).T
    assert np.array_equal(_bits(got), _bits(want))


def test_log_host_composes_the_line_passes():
    """log_host = sum over d = x, y, z of order 0 along the two other axes (x, y, z order) and order 2 along d."""
    rng = np.random.default_rng(5)
    v = rng.integers(-1000, 400, (5, 6, 7)).astype(np.int16)
    spacing, sigma = (0.7, 0.8, 1.25), 1.5
    f = v.astype(np.float64)

    def along(a, axis, order, s):
        c = lg.coefficients(sigma / s, order)
        out = np.empty_like(a)
        moved, res = np.moveaxis(a, axis, -1), np.moveaxis(out, axis, -1)
        for idx in np.ndindex(moved.shape[:-1]):
            res[idx] = _scalar_line(moved[idx], c)
        return out

    sx, sy, sz = spacing
    tx = along(along(along(f, 1, 0, sy), 0, 0, sz), 2, 2, sx)
    ty = along(along(along(f, 2, 0, sx), 0, 0, sz), 1, 2, sy)
    tz = along(along(along(f, 2, 0, sx), 1, 0, sy), 0, 2, sz)
    want = ((0.0 + tx) + ty) + tz
    assert np.array_equal(_bits(lg.log_host(v, sigma, spacing)), _bits(want))


# ---- independent properties ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("sd", [0.5, 1.0, 2.0, 5.0, 8.0])
def test_constant_line(sd):
    x = np.full((64, 1), -742.5)
    assert np.max(np.abs(lg.line_filter(x, lg.coefficients(sd, 0)) - x)) <= 1e-12 * 742.5
    assert np.max(np.abs(lg.line_filter(x, lg.coefficients(sd, 2)))) <= 1e-12 * 742.5


@pytest.mark.parametrize("sd", [1.0, 2.0, 3.0, 5.0, 8.0])
def test_second_derivative_of_a_parabola(sd):
    n = np.arange(601, dtype=np.float64) - 300
    x = ((n / sd) ** 2)[:, None]
    out = lg.line_filter(x, lg.coefficients(sd, 2))
    assert abs(out[300, 0] - 2.0) <= 1e-9


@pytest.mark.parametrize("sd", [1.0, 2.0, 3.0, 4.0, 5.0])
def test_impulse_responses_match_the_gaussian(sd):
    n = np.arange(201, dtype=np.float64) - 100
    x = np.zeros((201, 1))
    x[100] = 1.0
    g = np.exp(-n * n / (2 * sd * sd)) / (math.sqrt(2 * math.pi) * sd)
    h0 = lg.line_filter(x, lg.coefficients(sd, 0))[:, 0]
    assert np.max(np.abs(h0 - g)) <= 0.005 * g.max()
    g2 = g * (n * n / (sd * sd) - 1.0)            # sigma^2 G'' in samples
    h2 = lg.line_filter(x, lg.coefficients(sd, 2))[:, 0]
    assert np.max(np.abs(h2 - g2)) <= 0.02 * np.abs(g2).max()


@pytest.mark.parametrize("sigma", [1.0, 2.0, 3.0])
@pytest.mark.parametrize("spacing", [(1.0, 1.0, 1.0), (0.7, 0.7, 1.25), (1.0, 1.0, 2.5)])
def test_log_matches_scipy(sigma, spacing):
    from scipy import ndimage
    if sigma / max(spacing) < 0.8:
        pytest.skip("below 0.8 samples scipy's sampled second-derivative kernel is itself off (x^2 -> 2.65 at 0.4)")
    rng = np.random.default_rng(11)
    v = ndimage.gaussian_filter(rng.normal(0, 100, (40, 40, 40)), 1.5)
    s_arr = (spacing[2], spacing[1], spacing[0])       # per array axis (z, y, x)
    ref = np.zeros_like(v)
    for axis in range(3):
        order = [0, 0, 0]
        order[axis] = 2
        ref += sigma * sigma * ndimage.gaussian_filter(v, [sigma / s for s in s_arr], order=order, mode="nearest",
                                                       truncate=8.0) / (s_arr[axis] ** 2)
    got = lg.log_host(v, sigma, spacing)
    assert np.max(np.abs(got - ref)) <= 0.02 * np.max(np.abs(ref))


# ---- names, refusals, bin widths -----------------------------------------------------------------------------------

def test_names():
    assert lg.image_name(1) == "log-sigma-1-0-mm-3D"
    assert lg.image_name(2.5) == "log-sigma-2-5-mm-3D"
    assert lg.image_name(np.float32(3)) == "log-sigma-3-0-mm-3D"
    assert lg.check_sigmas([1, 2.5, 3]) == (1.0, 2.5, 3.0)
    assert lg.check_sigmas(2) == (2.0,)
    assert lg.parse_sigmas("1,2,3,4,5") == (1.0, 2.0, 3.0, 4.0, 5.0)


def test_refusals():
    for bad in ([], [0], [-1.0], [math.nan], [math.inf], [1, 1.0], [2.0, 1, 2]):
        with pytest.raises(ValueError):
            lg.check_sigmas(bad)
    for bad in ("1", [True], [None]):
        with pytest.raises(TypeError):
            lg.check_sigmas(bad)
    for bad in (None, (1, 0, 1), (1, 1), (1, -1, 1), (1, math.nan, 1)):
        with pytest.raises(ValueError):
            lg.check_spacing(bad)
    with pytest.raises(ValueError, match="under 4"):
        lg.check_shape((3, 10, 10))
    with pytest.raises(ValueError, match="2\\^32"):
        lg.check_shape((1 << 11, 1 << 11, 1 << 10))
    with pytest.raises(ValueError, match="sigma 5.0 mm .* along z"):
        lg.check_shape((5, 64, 64), (1.0, 1.0, 1.25), (5.0,))   # ceil(5 / 1.25) + 1 = 5 fits
        lg.check_shape((5, 64, 64), (1.0, 1.0, 1.0), (5.0,))    # ceil(5 / 1) + 1 = 6 does not
    lg.check_shape((6, 6, 6), (1.0, 1.0, 1.0), (5.0,))
    with pytest.raises(ValueError, match="along x"):
        lg.check_shape((6, 6, 5), (1.0, 1.0, 1.0), (4.5,))
    v = np.zeros((6, 6, 6))
    v[2, 3, 4] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        lg.log_host(v, 1.0, (1, 1, 1))
    with pytest.raises(ValueError):
        lg.log_host(np.zeros((6, 6, 6)), 1.0, None)


def test_bin_widths():
    sig = (1.0, 3.0)
    assert lg.check_bin_widths(25, sig) == {"log-sigma-1-0-mm-3D": 25, "log-sigma-3-0-mm-3D": 25}
    assert lg.check_bin_widths({1: 10, "log-sigma-3-0-mm-3D": 50, 5.0: 7}, sig) == \
        {"log-sigma-1-0-mm-3D": 10, "log-sigma-3-0-mm-3D": 50}
    with pytest.raises(ValueError, match="no bin width"):
        lg.check_bin_widths({1.0: 10}, sig)
    with pytest.raises(ValueError):
        lg.check_bin_widths(0, sig)
    assert lg.parse_bin_widths("25,3.0=50", sig) == {"log-sigma-1-0-mm-3D": 25, "log-sigma-3-0-mm-3D": 50}
    assert lg.parse_bin_widths("25", sig) == {"log-sigma-1-0-mm-3D": 25, "log-sigma-3-0-mm-3D": 25}
    for bad in ("x", "25,3.0=x", "25,30", "25,y=4", "3.0=50", "25,0=4"):
        with pytest.raises(ValueError):
            lg.parse_bin_widths(bad, sig)


def test_to_dict_keys():
    imgs = [lg.ImageFeatures(lg.image_name(s), 25) for s in (1.0, 2.0)]
    f = lg.LogFeatures((1.0, 2.0), ("firstorder",), (0.7, 0.7, 1.25), 0, 0, imgs)
    d = f.to_dict()
    assert d["sigmas"] == [1.0, 2.0]
    assert list(d["images"]) == ["log-sigma-1-0-mm-3D", "log-sigma-2-0-mm-3D"]
    assert f[2.0] is imgs[1] and f["log-sigma-1-0-mm-3D"] is imgs[0]


def test_abi_refuses_null_arguments():
    from lungmask_b200 import _native
    L = _native.lib()
    assert L.lm_laplacian_of_gaussian_dev(None, None, 0, 4, 4, 4, None, 1.0, None, None, None, None) == -1
    assert "NULL" in L.lm_last_error().decode()


# ---- CLI ---------------------------------------------------------------------------------------------------------------

def _cli_main(tmp_path, monkeypatch, argv):
    import lungmask_b200.__main__ as cli

    def no_load(*a, **k):
        raise AssertionError("the input was read before the arguments were checked")
    monkeypatch.setattr(cli, "load_input_image", no_load)
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    cli.main([str(src), str(tmp_path / "out.nii")] + argv)


@pytest.mark.parametrize("argv,msg", [
    (["--log", "l.json"], "--log: needs --log-sigma"),
    (["--texture", "t.json", "--log-sigma", "1"], "--log-sigma: needs --log"),
    (["--log", "l.json", "--log-sigma", "1,x"], "--log-sigma"),
    (["--log", "l.json", "--log-sigma", "0"], "--log-sigma"),
    (["--log", "l.json", "--log-sigma", "1,1.0"], "--log-sigma"),
    (["--log", "l.json", "--log-sigma", "1,2", "--log-bin-width", "25,x=4"], "--log-bin-width"),
    (["--log", "l.json", "--log-sigma", "1,2", "--log-bin-width", "0"], "--log-bin-width"),
    (["--log", "l.json", "--log-sigma", "1", "--log-classes", "glcm,foo"], "--log-classes"),
    (["--log", "l.txt", "--log-sigma", "1"], "unsupported log output format"),
])
def test_cli_refusals_before_segmentation(tmp_path, monkeypatch, argv, msg):
    argv = [str(tmp_path / a) if a.endswith((".json", ".txt")) else a for a in argv]
    with pytest.raises(SystemExit, match=msg):
        _cli_main(tmp_path, monkeypatch, argv)


def test_cli_log_arguments(tmp_path):
    from lungmask_b200.__main__ import build_parser, log_arguments, resample_arguments
    src = tmp_path / "in.npy"
    np.save(str(src), np.zeros((2, 2, 2), np.int16))
    args = build_parser().parse_args([str(src), "out.nii", "--log", "l.csv", "--log-sigma", "1,3",
                                      "--log-bin-width", "25,3.0=50", "--log-classes", "firstorder,glcm"])
    assert log_arguments(args) == ((1.0, 3.0), {"log-sigma-1-0-mm-3D": 25, "log-sigma-3-0-mm-3D": 50},
                                   ["firstorder", "glcm"])
    args = build_parser().parse_args([str(src), "out.nii", "--log", "l.json", "--log-sigma", "2", "--resample", "1,1,1"])
    assert log_arguments(args)[0] == (2.0,)
    assert resample_arguments(args) == ((1.0, 1.0, 1.0), "bspline")
    assert log_arguments(build_parser().parse_args([str(src), "out.nii"])) is None
