"""Device-resident volumes: LMInferer.apply / apply_with_probabilities / apply_oriented on CUDA tensors and the C entry
point behind them, lm_apply_dev.  Every result is compared bit for bit with the numpy path (or, for the fusion, with the
host entry points and a composition of stage entries); the input tensor must come back unchanged and the outputs live on
its device."""
import ctypes as C

import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

CODES = ["LPS", "RAS", "PLI", "SAL"]


def _direction(code):
    """Direction cosines (row-major 3x3) of an image whose axes x, y, z increase toward code[0], code[1], code[2]."""
    d = np.zeros((3, 3))
    for c, ch in enumerate(code):
        r = "LPS".index(ch) if ch in "LPS" else "RAI".index(ch)
        d[r, c] = 1.0 if ch in "LPS" else -1.0
    return tuple(d.ravel())


@pytest.fixture(scope="module")
def models():
    return {K: synth.random_state_dict(K, seed=10 + K, head_gain=0.3) for K in (3, 6)}


@pytest.fixture(scope="module")
def vol():
    """7 phantom slices at 200x216 plus one all-air slice (full-frame crop box), as in test_gpu_probabilities."""
    v = synth.phantom(7, 200, 216, seed=31)
    air = np.full((1, 200, 216), -1000, np.int16)
    return np.ascontiguousarray(np.concatenate([v[:4], air, v[4:]]))


@pytest.fixture(scope="module")
def weights(models, tmp_path_factory):
    import torch
    d = tmp_path_factory.mktemp("weights")
    paths = {K: str(d / ("w%d.pth" % K)) for K in models}
    for K, p in paths.items():
        torch.save(models[K], p)
    return paths


@pytest.fixture(scope="module")
def inf3(weights):
    from lungmask_b200 import LMInferer
    return LMInferer(modelpath=weights[3], batch_size=4, tqdm_disable=True)


@pytest.fixture(scope="module")
def inf_fused(weights):
    from lungmask_b200 import LMInferer
    return LMInferer(modelpath=weights[6], fillmodel="R231", fillmodel_path=weights[3], batch_size=4, tqdm_disable=True)


@pytest.fixture()
def fused_engine(engine, models):
    """The session engine with the fusion's two models: slot 0 = 6 classes (base), slot 1 = 3 classes (fill)."""
    from lungmask_b200.mask import NativeModel
    for slot, K in ((0, 6), (1, 3)):
        m = NativeModel(models[K])
        engine.load_weights(slot, m.blob, m.n_classes)
    return engine


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _checked(fn, t):
    """fn(t); asserts that t is unchanged and that every returned tensor lives on t's device."""
    before = t.clone()
    res = fn(t)
    import torch
    assert torch.equal(t, before), "the input tensor was modified"
    for r in res if isinstance(res, tuple) else (res,):
        assert r is None or r.device == t.device
    return res


def _np(t):
    return t.cpu().numpy()


def _dev(engine, slot, t, code="LPS", slot_fill=-1, probs=False, postprocess=True):
    """engine.apply_dev on a CUDA tensor (native orientation `code`) -> (mask, probs or None) as tensors."""
    import torch
    from lungmask_b200 import orient
    from lungmask_b200.mask import _tensor_dtype_code
    perm, flip = (None, None) if code == "LPS" else orient.array_transform_to_lps(code)
    out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    p = torch.empty((engine.n_classes[slot],) + tuple(t.shape), dtype=torch.float32, device=t.device) if probs else None
    engine.apply_dev(slot, t.data_ptr(), _tensor_dtype_code(t), t.shape, out.data_ptr(), perm, flip, slot_fill=slot_fill,
                     d_probs_ptr=p.data_ptr() if p is not None else None, postprocess=postprocess,
                     stream=torch.cuda.current_stream().cuda_stream)
    return out, p


@pytest.mark.parametrize("dtype", [np.int16, np.float32, np.float64])
@pytest.mark.parametrize("code", CODES)
def test_mask_equals_numpy_path(inf3, vol, dtype, code):
    import torch
    from lungmask_b200 import orient
    v = vol if dtype == np.int16 else (vol.astype(np.float64) + 0.375).astype(dtype)
    native = orient.from_lps(v, code)
    t = _cuda(native)
    try:
        for pp in (True, False):
            inf3.volume_postprocessing = pp
            want = inf3.apply_oriented(native, _direction(code))
            got = _checked(lambda x: inf3.apply_oriented(x, _direction(code)), t)
            assert got.dtype == torch.uint8 and tuple(got.shape) == native.shape
            assert np.array_equal(_np(got), want), (pp, code)
            if code == "LPS":
                assert np.array_equal(_np(_checked(inf3.apply, t)), want)
    finally:
        inf3.volume_postprocessing = True


@pytest.mark.parametrize("K", [3, 6])
@pytest.mark.parametrize("code", ["LPS", "PLI"])
def test_probabilities_equal_numpy_path(engine, models, vol, K, code):
    from lungmask_b200 import orient
    from lungmask_b200.mask import NativeModel
    m = NativeModel(models[K])
    engine.load_weights(0, m.blob, m.n_classes)
    perm, flip = (None, None) if code == "LPS" else orient.array_transform_to_lps(code)
    for v in (vol, (vol.astype(np.float64) + 0.375).astype(np.float32)):
        native = orient.from_lps(v, code)
        want_m, want_p = engine.apply_volume_probs(0, native, perm, flip)
        got_m, got_p = _checked(lambda x: _dev(engine, 0, x, code, probs=True), _cuda(native))
        assert got_p.dtype.is_floating_point and tuple(got_p.shape) == (K,) + native.shape
        assert np.array_equal(_np(got_m), want_m)
        assert np.array_equal(_np(got_p), want_p)


def test_apply_with_probabilities_tensor(inf3, vol):
    import torch
    want_m, want_p = inf3.apply_with_probabilities(vol)
    got_m, got_p = _checked(inf3.apply_with_probabilities, _cuda(vol))
    assert got_m.dtype == torch.uint8 and got_p.dtype == torch.float32
    assert np.array_equal(_np(got_m), want_m) and np.array_equal(_np(got_p), want_p)
    cpu_m, cpu_p = inf3.apply_with_probabilities(torch.from_numpy(vol))   # CPU tensor: the numpy path, CPU tensors back
    assert cpu_m.device.type == "cpu" and np.array_equal(cpu_m.numpy(), want_m) and np.array_equal(cpu_p.numpy(), want_p)


@pytest.mark.parametrize("code", ["LPS", "SAL"])
def test_fusion_int16(fused_engine, inf_fused, vol, code):
    from lungmask_b200 import orient
    eng = fused_engine
    native = orient.from_lps(vol, code)
    t = _cuda(native)
    for pp in (True, False):
        if code == "LPS":
            want = eng.apply_fused(0, 1, native, postprocess=pp)
        else:
            perm, flip = orient.array_transform_to_lps(code)
            want = eng.apply_volume_oriented(0, native, perm, flip, slot_fill=1, postprocess=pp)
        got, _ = _checked(lambda x: _dev(eng, 0, x, code, slot_fill=1, postprocess=pp), t)
        assert np.array_equal(_np(got), want), (code, pp)
        inf_fused.volume_postprocessing = pp
        try:
            assert np.array_equal(_np(_checked(lambda x: inf_fused.apply_oriented(x, _direction(code)), t)), want)
        finally:
            inf_fused.volume_postprocessing = True


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("code", ["LPS", "PLI", "SAL"])
def test_fusion_float_any_orientation(fused_engine, inf_fused, vol, dtype, code):
    """The fusion of a float volume in any orientation (LMInferer raised NotImplementedError for non-LPS before) equals
    the reference's sequence written with stage entries: per model the float path on the LPS array, each result back in
    the native orientation, the spare-label fusion there and its post-processing."""
    from lungmask_b200 import orient
    eng = fused_engine
    v = (vol.astype(np.float64) + 0.375).astype(dtype)
    native = orient.from_lps(v, code)
    res = [orient.from_lps(eng.apply_volume_float(s, orient.to_lps(native, code)), code) for s in (0, 1)]
    fused, spare = eng.fuse(res[0], res[1])
    want = eng.postprocess(fused, spare=[spare])
    got, _ = _checked(lambda x: _dev(eng, 0, x, code, slot_fill=1), _cuda(native))
    assert np.array_equal(_np(got), want)
    assert np.array_equal(inf_fused.apply_oriented(native, _direction(code)), want)      # the host path
    assert np.array_equal(_np(_checked(lambda x: inf_fused.apply_oriented(x, _direction(code)), _cuda(native))), want)


def test_other_dtypes(inf3, vol):
    import torch
    from lungmask_b200 import orient
    wide = vol.astype(np.int64)
    wide[:, 10:30, 20:40] = 40000                    # outside int16: the clip to [-1024, 600] must come first
    wide[:, 150:170, 100:140] = -40000
    arrays = {"bool": vol > -500, "uint8": np.clip(vol, 0, 255).astype(np.uint8),
              "int8": np.clip(vol, -128, 127).astype(np.int8), "int32": wide.astype(np.int32), "int64": wide}
    for name, a in arrays.items():
        want = inf3.apply(a)
        assert np.array_equal(_np(_checked(inf3.apply, _cuda(a))), want), name
    native = orient.from_lps(arrays["int32"], "PLI")          # conversion and re-orientation in one pass
    want = inf3.apply_oriented(native, _direction("PLI"))
    assert np.array_equal(_np(_checked(lambda x: inf3.apply_oriented(x, _direction("PLI")), _cuda(native))), want)

    vf = torch.from_numpy((vol.astype(np.float64) + 0.375).astype(np.float32))
    for dt in (torch.float16, torch.bfloat16):
        t = vf.to(dt)
        want = inf3.apply(t.float().numpy())
        assert np.array_equal(_np(_checked(inf3.apply, t.to("cuda:0"))), want), dt
        assert np.array_equal(inf3.apply(t).numpy(), want), dt         # CPU tensor
        want_m, want_p = inf3.apply_with_probabilities(t.float().numpy())
        got_m, got_p = inf3.apply_with_probabilities(t.to("cuda:0"))
        assert np.array_equal(_np(got_m), want_m) and np.array_equal(_np(got_p), want_p), dt


def test_float16_warns(inf3, vol, caplog):
    import torch
    t = torch.from_numpy(vol.astype(np.float32)).to("cuda:0", torch.float16)
    with caplog.at_level("WARNING", logger="lungmask"):
        inf3.apply(t)
    assert any("float32" in r.getMessage() for r in caplog.records)


def test_noncontiguous_input(inf3, vol):
    t = _cuda(np.ascontiguousarray(vol.transpose(0, 2, 1))).transpose(1, 2)    # a strided view of vol
    assert not t.is_contiguous()
    assert np.array_equal(_np(_checked(inf3.apply, t)), inf3.apply(vol))


def test_stream_ordering(inf3, vol):
    """The producer of the volume is still running (a ~1e8-cycle sleep, then the copy) when apply is called: the engine
    must wait for it on the caller's stream, with no synchronisation by the caller."""
    import torch
    want = inf3.apply(vol)
    src = _cuda(vol)
    side = torch.cuda.Stream(device=0)
    for use_side in (True, False):
        t = torch.full(vol.shape, -1000, dtype=torch.int16, device="cuda:0")
        torch.cuda.synchronize()
        stream = side if use_side else torch.cuda.default_stream(0)
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)
            t.copy_(src)
            got = inf3.apply(t)
        assert np.array_equal(_np(got), want), "side stream" if use_side else "default stream"
        torch.cuda.synchronize()


def test_errors(fused_engine, inf3, inf_fused, vol):
    import torch
    from lungmask_b200 import _native
    t = _cuda(vol)
    with pytest.raises(ValueError, match="slices, H, W"):
        inf3.apply(t[0])
    with pytest.raises(TypeError, match="dtype"):
        inf3.apply(t.to(torch.complex64))
    with pytest.raises(TypeError, match="dtype"):
        inf3.apply(torch.empty(vol.shape, dtype=torch.uint16, device="cuda:0"))
    with pytest.raises(ValueError, match="meta"):
        inf3.apply(torch.empty(vol.shape, dtype=torch.int16, device="meta"))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="engine"):
            inf3.apply(t.to("cuda:1"))
    with pytest.raises(ValueError, match="fill model"):
        inf_fused.apply_with_probabilities(t)

    eng = fused_engine
    L = _native.lib()
    out = torch.empty(vol.shape, dtype=torch.uint8, device="cuda:0")
    probs = torch.empty((6,) + vol.shape, dtype=torch.float32, device="cuda:0")
    n0, n1, n2 = vol.shape

    def raw(d_vol, dtype, slot_fill=-1, d_probs=None):
        return L.lm_apply_dev(eng._h, 0, slot_fill, C.c_void_p(d_vol), dtype, n0, n1, n2, None, None, 0,
                              C.c_void_p(out.data_ptr()), C.c_void_p(d_probs) if d_probs else None, None)

    rc = raw(t.data_ptr(), _native.DTYPE_I16, slot_fill=1, d_probs=probs.data_ptr())
    assert rc != 0 and "fusion" in L.lm_last_error().decode()
    rc = raw(t.data_ptr(), 9)
    assert rc != 0 and "dtype" in L.lm_last_error().decode()
    pinned = torch.from_numpy(vol).pin_memory()                 # host memory is refused before any kernel reads it
    rc = raw(pinned.data_ptr(), _native.DTYPE_I16)
    assert rc != 0 and "device memory" in L.lm_last_error().decode()
    with pytest.raises(_native.NativeError, match="permutation"):
        eng.apply_dev(0, t.data_ptr(), _native.DTYPE_I16, vol.shape, out.data_ptr(), perm=(0, 0, 1), flip=(0, 0, 0))
    with pytest.raises(_native.NativeError, match="not loaded"):      # inf3 has no fill model: its slot 1 is empty
        inf3.engine.apply_dev(1, t.data_ptr(), _native.DTYPE_I16, vol.shape, out.data_ptr())
    with pytest.raises(_native.NativeError, match="empty"):
        eng.apply_dev(0, t.data_ptr(), _native.DTYPE_I16, (0, n1, n2), out.data_ptr())
