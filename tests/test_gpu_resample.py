"""Resampling on the GPU (LMInferer.resample; lm_bspline_coefficients_dev, lm_resample_dev) against the numpy statement
lungmask_b200.resample: the coefficient volume as uint64 bit patterns for every dtype code, odd and even extents,
extents of 1, 2, 18 and 19 and the 300x512x512 phantom; the resampled image and mask bit for bit for both
interpolators, every dtype, up- and downsampling, anisotropic targets, the crop-only case and every input kind; the
refusals; and --resample on the command line against the same chain in Python."""
import os

import numpy as np
import pytest

from lungmask_b200 import _native
from lungmask_b200 import resample as rsm
from oracle import synth

pytestmark = pytest.mark.gpu

SPACING = (0.7, 0.8, 2.5)   # (x, y, z) mm


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


def _host(a):
    """A result as a numpy array (bfloat16 tensors as their uint16 bit patterns)."""
    import torch
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu()
        if a.dtype == torch.bfloat16:
            return a.view(torch.int16).numpy().view(np.uint16)
        return a.numpy()
    return np.asarray(a)


def same_bits(got, want):
    got, want = _host(got), _host(want)
    return got.shape == want.shape and got.dtype == want.dtype and np.array_equal(
        np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def two_lungs(S, H, W):
    z, y, x = np.ogrid[:S, :H, :W]
    m = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        m[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    return m


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
    x.view(-1)[:2] = torch.tensor([0.0, -0.0], dtype=torch.float64)[:x.numel()]
    return x.to(dtype)


def _coefficients(inf, t):
    import torch
    from lungmask_b200.mask import _tensor_dtype_code
    t = t.cuda().contiguous()
    out = torch.empty(tuple(t.shape), dtype=torch.float64, device=t.device)
    inf.engine.bspline_coefficients_dev(t.data_ptr(), _tensor_dtype_code(t), t.shape, out.data_ptr())
    return out.cpu().numpy()


ALL_DTYPES = ("uint8", "int8", "int16", "int32", "int64", "float16", "bfloat16", "float32", "float64", "bool")


# ---- coefficients

def test_coefficients_every_dtype_code(inf):
    import torch
    for k, name in enumerate(ALL_DTYPES):
        t = _values(getattr(torch, name), (7, 10, 37), 300 + k)
        got = _coefficients(inf, t)
        assert np.array_equal(got.view(np.uint64), rsm.decompose_host(t.double().numpy()).view(np.uint64)), name


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 1, 19), (18, 19, 2), (19, 18, 1), (1, 2, 18), (3, 33, 32),
                                   (5, 64, 65), (20, 7, 100)])
def test_coefficients_extents(inf, shape):
    import torch
    t = _values(torch.float32, shape, sum(shape))
    assert np.array_equal(_coefficients(inf, t).view(np.uint64), rsm.decompose_host(t.double().numpy()).view(np.uint64))
    t = _values(torch.int16, shape, sum(shape) + 1)
    assert np.array_equal(_coefficients(inf, t).view(np.uint64), rsm.decompose_host(t.double().numpy()).view(np.uint64))


# ---- resampled image and mask

CASES = [   # resampled spacing, pad
    ((1.0, 1.0, 1.0), 5),    # in-plane down, z up
    ((0.5, 0.45, 0.6), 2),   # up on every axis
    ((2.0, 1.5, 0.0), 1),    # down, z kept
    ((1.3, 0.6, 3.1), 0),    # anisotropic, pad 0
    (SPACING, 3),            # crop only
]


def _pair(shape, seed, dtype=np.int16):
    rng = np.random.default_rng(seed)
    vol = rng.integers(-1024, 1500, shape).astype(dtype)
    mask = np.zeros(shape, np.uint8)
    S, H, W = shape
    mask[1:S - 1, 2:H - 3, 3:W - 1] = rng.integers(0, 4, (S - 2, H - 5, W - 4))
    return vol, mask


@pytest.mark.parametrize("interpolator", ["bspline", "nearest"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_resample_matches_statement(inf, interpolator, case):
    rs, pad = CASES[case]
    vol, mask = _pair((9, 22, 27), 40 + case)
    r = inf.resample(vol, mask, rs, spacing=SPACING, interpolator=interpolator, pad_distance=pad)
    img, m, g = rsm.resample_host(vol, mask, SPACING, rs, interpolator, pad)
    assert same_bits(r.image, img) and same_bits(r.mask, m)
    assert r.spacing == g.spacing and r.start == g.start
    assert r.origin is None and r.direction is None


@pytest.mark.parametrize("interpolator", ["bspline", "nearest"])
def test_resample_every_dtype(inf, interpolator):
    import torch
    shape = (6, 17, 20)
    mask = _pair(shape, 1)[1]
    for k, name in enumerate(ALL_DTYPES[:-1]):
        t = _values(getattr(torch, name), shape, 500 + k)
        ref = t.float().numpy() if name == "bfloat16" else t.numpy()
        img, m, _ = rsm.resample_host(ref, mask, SPACING, (1.1, 0.5, 1.0), interpolator, 2)
        want = torch.from_numpy(img).to(torch.bfloat16) if name == "bfloat16" else img
        got = inf.resample(t.cuda(), _cuda(mask), (1.1, 0.5, 1.0), spacing=SPACING, interpolator=interpolator,
                           pad_distance=2)
        assert got.image.is_cuda and got.image.dtype == t.dtype, name
        assert same_bits(got.image, want) and same_bits(got.mask, m), (name, "cuda")
        got = inf.resample(t, torch.from_numpy(mask), (1.1, 0.5, 1.0), spacing=SPACING, interpolator=interpolator,
                           pad_distance=2)
        assert not got.image.is_cuda and got.image.dtype == t.dtype, name
        assert same_bits(got.image, want) and same_bits(got.mask, m), (name, "cpu tensor")
    for dtype in (np.uint16, np.uint32):   # widened for the device, narrowed back with the same clamp
        v = np.random.default_rng(9).integers(0, 3000, shape).astype(dtype)
        got = inf.resample(v, mask, (1.1, 0.5, 1.0), spacing=SPACING, interpolator=interpolator)
        assert same_bits(got.image, rsm.resample_host(v, mask, SPACING, (1.1, 0.5, 1.0), interpolator)[0]), dtype


def test_crop_only_keeps_values(inf):
    vol, mask = _pair((9, 22, 27), 3, np.float32)
    r = inf.resample(vol, mask, SPACING, spacing=SPACING, pad_distance=1)
    lo, size = rsm.bounding_box(mask)
    sl = tuple(slice(max(lo[d] - 1, 0), min(lo[d] + size[d] + 1, vol.shape[2 - d])) for d in (2, 1, 0))
    assert same_bits(r.image, vol[sl]) and same_bits(r.mask, mask[sl])
    assert r.spacing == SPACING


def test_input_kinds_and_geometry(inf):
    import torch
    from lungmask_b200.io import Volume
    vol, mask = _pair((11, 30, 25), 8)
    want_img, want_m, g = rsm.resample_host(vol, mask, SPACING, (1.0, 1.0, 1.0))
    D = (0.0, 1.0, 0.0, -1.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    v = Volume(vol, SPACING, (-10.0, 20.5, 3.0), D)
    r = inf.resample(v, mask)
    assert isinstance(r.image, np.ndarray) and same_bits(r.image, want_img) and same_bits(r.mask, want_m)
    assert r.direction == D and r.origin == rsm.new_origin((-10.0, 20.5, 3.0), D, SPACING, g.start)
    rv = r.volume()
    assert rv.spacing == g.spacing and rv.origin == r.origin and rv.direction == D and rv.array is r.image
    tv, tm = _cuda(vol), _cuda(mask)
    r = inf.resample(tv, tm, spacing=SPACING)
    assert r.image.is_cuda and r.mask.is_cuda and same_bits(r.image, want_img) and same_bits(r.mask, want_m)
    assert np.array_equal(tv.cpu().numpy(), vol) and np.array_equal(tm.cpu().numpy(), mask)
    r = inf.resample(torch.from_numpy(vol), torch.from_numpy(mask), spacing=SPACING)
    assert isinstance(r.image, torch.Tensor) and not r.image.is_cuda and same_bits(r.image, want_img)
    # the result feeds the feature calls as they are
    t = inf.texture(r.image.numpy(), r.mask.numpy(), spacing=r.spacing)
    assert t.spacing == g.spacing


def test_cuda_inputs_read_after_work_on_the_callers_stream(inf):
    import torch
    vol, mask = _pair((9, 22, 27), 12)
    want_img, want_m, _ = rsm.resample_host(vol, mask, SPACING, (1.0, 1.0, 1.0))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        tv = torch.zeros(vol.shape, dtype=torch.int16, device="cuda:0")
        tm = torch.zeros(mask.shape, dtype=torch.uint8, device="cuda:0")
        torch.cuda._sleep(50_000_000)
        tv.copy_(torch.from_numpy(vol).cuda(non_blocking=False))
        tm.copy_(torch.from_numpy(mask).cuda(non_blocking=False))
        r = inf.resample(tv, tm, spacing=SPACING)
    assert same_bits(r.image, want_img) and same_bits(r.mask, want_m)


def test_300x512x512_phantom(inf):
    """The coefficient volume of the int16 phantom bit for bit; the whole mask and 6 output planes (first and last
    included) of the image."""
    import torch
    vol = synth.phantom(300, 512, 512, seed=31)
    mask = two_lungs(300, 512, 512)
    sp = (0.703125, 0.703125, 1.25)
    tv, tm = _cuda(vol), _cuda(mask)
    coeff = torch.empty(vol.shape, dtype=torch.float64, device="cuda:0")
    inf.engine.bspline_coefficients_dev(tv.data_ptr(), _native.DTYPE_I16, vol.shape, coeff.data_ptr())
    want_coeff = rsm.decompose_host(vol)
    assert np.array_equal(coeff.cpu().numpy().view(np.uint64), want_coeff.view(np.uint64))
    del coeff
    r = inf.resample(tv, tm, (1.0, 1.0, 1.0), spacing=sp)
    g = rsm.grid(vol.shape, sp, (1.0, 1.0, 1.0), *rsm.bounding_box(mask))
    M = g.shape[0]
    planes = np.array(sorted({0, 1, M // 3, M // 2, M - 2, M - 1}))
    img, m, _ = rsm.resample_host(vol, mask, sp, (1.0, 1.0, 1.0), planes=planes, coeff=want_coeff)
    assert tuple(r.image.shape) == g.shape
    assert same_bits(r.image[torch.from_numpy(planes).cuda()], img)
    _, m_all, _ = rsm.resample_host(vol, mask, sp, (1.0, 1.0, 1.0), interpolator="nearest")
    assert same_bits(r.mask, m_all)
    assert np.array_equal(tv.cpu().numpy(), vol)


# ---- refusals

def test_refusals(inf):
    import torch
    vol, mask = _pair((6, 10, 12), 2, np.float32)
    bad = vol.copy()
    bad[2, 3, 4] = np.nan
    for interp in ("bspline", "nearest"):
        with pytest.raises(ValueError, match="NaN"):
            inf.resample(bad, mask, spacing=SPACING, interpolator=interp)
        with pytest.raises(ValueError, match="NaN"):
            inf.resample(_cuda(bad), _cuda(mask), spacing=SPACING, interpolator=interp)
    with pytest.raises(ValueError, match="empty"):
        inf.resample(vol, np.zeros_like(mask), spacing=SPACING)
    with pytest.raises(ValueError, match="spacing"):
        inf.resample(vol, mask)
    with pytest.raises(ValueError, match="pad_distance"):
        inf.resample(vol, mask, spacing=SPACING, pad_distance=-1)
    with pytest.raises(ValueError, match="shape"):
        inf.resample(vol, mask[:, :, :5], spacing=SPACING)
    with pytest.raises(ValueError, match="2\\^32"):
        inf.resample(vol, mask, (1e-3, 1e-3, 1e-3), spacing=SPACING)
    with pytest.raises(TypeError, match="bool"):
        inf.resample(vol > 0, mask, spacing=SPACING)
    # the C ABI: overlapping buffers, a non-finite table, no coefficients for the B-spline
    tv, tm = _cuda(vol), _cuda(mask)
    tab = torch.zeros(4, dtype=torch.float64, device="cuda:0")
    out = torch.empty((4, 4, 4), dtype=torch.float32, device="cuda:0")
    om = torch.empty((4, 4, 4), dtype=torch.uint8, device="cuda:0")
    e = inf.engine
    code = _native.DTYPE_F32
    ptrs = [tab.data_ptr()] * 3
    with pytest.raises(ValueError, match="overlaps"):
        e.resample_dev(tv.data_ptr(), code, None, tm.data_ptr(), vol.shape, ptrs, (4, 4, 4), "nearest", tv.data_ptr(),
                       om.data_ptr())
    with pytest.raises(ValueError, match="overlaps"):
        e.resample_dev(tv.data_ptr(), code, None, tm.data_ptr(), vol.shape, ptrs, (4, 4, 4), "nearest", out.data_ptr(),
                       out.data_ptr())
    with pytest.raises(ValueError, match="overlaps"):
        e.bspline_coefficients_dev(tv.data_ptr(), code, vol.shape, tv.data_ptr())
    with pytest.raises(ValueError, match="d_coeff"):
        e.resample_dev(tv.data_ptr(), code, None, tm.data_ptr(), vol.shape, ptrs, (4, 4, 4), "bspline", out.data_ptr(),
                       om.data_ptr())
    tab[1] = float("inf")
    with pytest.raises(ValueError, match="NaN"):
        e.resample_dev(tv.data_ptr(), code, None, tm.data_ptr(), vol.shape, ptrs, (4, 4, 4), "nearest", out.data_ptr(),
                       om.data_ptr())
    # the engine still works after the refusals
    r = inf.resample(vol, mask, spacing=SPACING)
    assert same_bits(r.image, rsm.resample_host(vol, mask, SPACING)[0])


# ---- command line

def test_cli_resample_equals_python_chain(tmp_path):
    import torch
    from lungmask_b200 import LMInferer
    from lungmask_b200.__main__ import main
    from lungmask_b200.io import Volume, _write_mha, load_input_image, save_shape, save_texture
    p = str(tmp_path / "w.pth")
    torch.save(synth.random_state_dict(3, seed=13, head_gain=0.3), p)
    src = str(tmp_path / "vol.mha")
    vol = synth.phantom(12, 96, 96, seed=21)
    _write_mha(src, vol, Volume(vol, (0.7, 0.7, 2.5), (1.0, -2.0, 3.0)))
    T, S = str(tmp_path / "t.json"), str(tmp_path / "s.json")
    main([src, str(tmp_path / "m.npy"), "--modelpath", p, "--noprogress", "--resample", "1,1,1", "--texture", T,
          "--shape", S])
    inferer = LMInferer(modelpath=p, tqdm_disable=True)
    image = load_input_image(src)
    result = inferer.apply(image)
    r = inferer.resample(image, result, (1, 1, 1))
    assert r.spacing == (1.0, 1.0, 1.0) and r.image.shape != vol.shape
    T2, S2 = str(tmp_path / "t2.json"), str(tmp_path / "s2.json")
    save_texture(T2, inferer.texture(r.volume(), r.mask))
    save_shape(S2, inferer.shape(r.mask, image=r.volume()))
    assert open(T).read() == open(T2).read()
    assert open(S).read() == open(S2).read()
