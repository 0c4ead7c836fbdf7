"""The whole-volume entry points share one path: for the same volume, every host, device and oriented variant of a call
returns the same mask bit for bit, and the host and device variants launch the same number of kernels.  The volume is
not a multiple of 256 in-plane and spans three waves of the engine's batch."""
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

BASE, FILL, EMPTY = 0, 1, 2        # weight slots: the 6-class base model, the 3-class fill model, never loaded
SLOT_OF_K = {6: BASE, 3: FILL}
IDENTITY = dict(perm=(0, 1, 2), flip=(0, 0, 0))


@pytest.fixture(scope="module")
def eng():
    from lungmask_b200 import _native
    from lungmask_b200.mask import NativeModel
    e = _native.Engine(device=0, batch_capacity=4)
    for K, slot in SLOT_OF_K.items():
        m = NativeModel(synth.random_state_dict(K, seed=20 + K, head_gain=0.3))
        e.load_weights(slot, m.blob, m.n_classes)
    yield e
    e.close()


@pytest.fixture(scope="module")
def vol():
    """10 phantom slices at 200x216 plus one all-air slice (full-frame crop box)."""
    v = synth.phantom(10, 200, 216, seed=41)
    air = np.full((1, 200, 216), -1000, np.int16)
    return np.ascontiguousarray(np.concatenate([v[:6], air, v[6:]]))


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _on_device(call, t):
    """call(d_vol_ptr, d_out_ptr) on the CUDA tensor t -> the mask as a numpy array."""
    import torch
    out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    torch.cuda.synchronize()       # lm_apply_volume_dev / lm_apply_fused_dev leave the ordering of their input to the caller
    call(t.data_ptr(), out.data_ptr())
    return out.cpu().numpy()


def _launches(eng):
    return eng.last_timings()["kernel_launches"]


@pytest.mark.parametrize("postprocess", [True, False])
@pytest.mark.parametrize("K", [3, 6])
def test_single_model(eng, vol, K, postprocess):
    from lungmask_b200 import _native
    slot, t = SLOT_OF_K[K], _cuda(vol)
    want = eng.apply_volume(slot, vol, postprocess=postprocess)
    host_launches = _launches(eng)
    got = _on_device(lambda v, o: eng.apply_volume_dev(slot, v, vol.shape, o, postprocess=postprocess), t)
    assert np.array_equal(got, want)
    assert _launches(eng) == host_launches
    got = _on_device(lambda v, o: eng.apply_dev(slot, v, _native.DTYPE_I16, vol.shape, o, postprocess=postprocess), t)
    assert np.array_equal(got, want)
    assert np.array_equal(eng.apply_volume_oriented(slot, vol, postprocess=postprocess, **IDENTITY), want)
    mask, probs = eng.apply_volume_probs(slot, vol, postprocess=postprocess)
    assert np.array_equal(mask, want)
    assert probs.shape == (K,) + vol.shape


@pytest.mark.parametrize("postprocess", [True, False])
def test_fusion(eng, vol, postprocess):
    from lungmask_b200 import _native
    t = _cuda(vol)
    want = eng.apply_fused(BASE, FILL, vol, postprocess=postprocess)
    host_launches = _launches(eng)
    got = _on_device(lambda v, o: eng.apply_fused_dev(BASE, FILL, v, vol.shape, o, postprocess=postprocess), t)
    assert np.array_equal(got, want)
    assert _launches(eng) == host_launches
    assert np.array_equal(eng.apply_volume_oriented(BASE, vol, slot_fill=FILL, postprocess=postprocess, **IDENTITY), want)
    got = _on_device(lambda v, o: eng.apply_dev(BASE, v, _native.DTYPE_I16, vol.shape, o, slot_fill=FILL,
                                                postprocess=postprocess), t)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("postprocess", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float(eng, vol, dtype, postprocess):
    from lungmask_b200 import _native
    v = (vol.astype(np.float64) + 0.375).astype(dtype)
    t = _cuda(v)
    code = _native.DTYPE_F32 if dtype == np.float32 else _native.DTYPE_F64
    for slot, fill in ((BASE, -1), (FILL, -1), (BASE, FILL)):
        want = eng.apply_volume_float(slot, v, slot_fill=fill, postprocess=postprocess)
        host_launches = _launches(eng)
        got = _on_device(lambda a, o: eng.apply_dev(slot, a, code, v.shape, o, slot_fill=fill, postprocess=postprocess), t)
        assert np.array_equal(got, want), (slot, fill)
        assert _launches(eng) == host_launches, (slot, fill)


def test_fused_needs_a_fill_model(eng, vol):
    """slot_fill < 0 does not fall back to the base model's mask: like a fill slot that holds no weights, it is refused."""
    import torch
    from lungmask_b200 import _native
    t = _cuda(vol)
    out = torch.empty(vol.shape, dtype=torch.uint8, device=t.device)
    for fill in (-1, EMPTY):
        with pytest.raises(_native.NativeError, match="not loaded"):
            eng.apply_fused(BASE, fill, vol)
        with pytest.raises(_native.NativeError, match="not loaded"):
            eng.apply_fused_dev(BASE, fill, t.data_ptr(), vol.shape, out.data_ptr())
    assert np.array_equal(eng.apply_fused(BASE, FILL, vol), eng.apply_volume_oriented(BASE, vol, slot_fill=FILL, **IDENTITY))
