"""LMInferer.apply_with_probabilities / lm_apply_volume_probs: the mask of `apply` plus the per-class probabilities
exp(log-softmax) of the same forward pass, resampled to the input like the mask (order 0 into the crop box, class 0
with certainty where the mask resampling writes 0) and returned in the input's own orientation."""
import ctypes as C
import struct
import gzip

import numpy as np
import pytest

from oracle import restate, synth

pytestmark = pytest.mark.gpu

TOL_P = 1e-4   # the scores match the reference within 1e-4 and d exp(s) / ds <= 1 for s <= 0


def _blob(sd):
    from lungmask_b200.mask import NativeModel
    return NativeModel(sd)


@pytest.fixture(scope="module")
def models():
    return {K: synth.random_state_dict(K, seed=10 + K, head_gain=0.3) for K in (3, 6)}


@pytest.fixture(scope="module")
def vol():
    """7 phantom slices at 200x216 plus one all-air slice: its crop box is the whole frame, where the order-0 zoom from
    256 leaves a zero last row and column (scipy's constant mode).  8 slices = waves of 4 + 4 on the session engine;
    the float tests and the orientation tests also run 200 / 216-slice permutations of it."""
    v = synth.phantom(7, 200, 216, seed=31)
    air = np.full((1, 200, 216), -1000, np.int16)
    return np.ascontiguousarray(np.concatenate([v[:4], air, v[4:]]))


def _load(engine, models, K):
    m = _blob(models[K])
    engine.load_weights(0, m.blob, m.n_classes)


def _expected(vol, sd):
    """numpy statement of the contract: exp of the oracle's scores, order-0 zoom into each slice's box, one-hot class 0
    wherever utils.reshape_mask of an all-ones mask gives 0."""
    taps = {}
    restate.inference(vol, sd, batch_size=4, volume_postprocessing=False, taps=taps)
    scores, boxes = taps["scores"], taps["boxes"]
    K, (S, H, W) = scores.shape[1], vol.shape
    want = np.zeros((K, S, H, W), np.float32)
    for s in range(S):
        b = boxes[s]
        (cy, _), (cx, _) = restate.zoom_src_coord(256, b[2] - b[0]), restate.zoom_src_coord(256, b[3] - b[1])
        iy = np.clip(np.floor(cy + 0.5).astype(np.int64), 0, 255)
        ix = np.clip(np.floor(cx + 0.5).astype(np.int64), 0, 255)
        want[:, s, b[0]:b[2], b[1]:b[3]] = np.exp(scores[s])[:, iy][:, :, ix]
        zero = restate.reshape_mask(np.ones((256, 256), np.uint8), b, (H, W)) == 0
        want[0, s][zero] = 1.0
        want[1:, s][:, zero] = 0.0
    return want, boxes


@pytest.mark.parametrize("K", [3, 6])
def test_probabilities_oracle(engine, models, vol, K):
    _load(engine, models, K)
    mask, probs = engine.apply_volume_probs(0, vol, postprocess=False)
    want, boxes = _expected(vol, models[K])
    assert tuple(boxes[4]) == (0, 0, 200, 216)                  # the all-air slice: full-frame box
    assert probs.dtype == np.float32 and probs.shape == (K,) + vol.shape
    err = np.abs(probs - want)
    print("K=%d max|dp|=%.3e mean=%.3e" % (K, err.max(), err.mean()))
    assert err.max() <= TOL_P
    assert np.all(probs[0, 4, -1, :] == 1.0) and np.all(probs[0, 4, :, -1] == 1.0)   # the quirk row / column
    assert np.abs(probs.sum(0, dtype=np.float64) - 1.0).max() <= 1e-5


@pytest.mark.parametrize("postprocess", [True, False])
def test_mask_identity(engine, models, vol, postprocess):
    _load(engine, models, 6)
    mask, _ = engine.apply_volume_probs(0, vol, postprocess=postprocess)
    assert np.array_equal(mask, engine.apply_volume(0, vol, postprocess=postprocess))


@pytest.mark.parametrize("K", [3, 6])
def test_argmax_identity(engine, models, vol, K):
    _load(engine, models, K)
    mask, probs = engine.apply_volume_probs(0, vol, postprocess=False)
    top2 = np.sort(probs, axis=0)[-2:]
    decided = (top2[1] - top2[0]) > 1e-6
    print("K=%d near-ties (top-2 within 1e-6): %d of %d voxels" % (K, (~decided).sum(), decided.size))
    assert np.array_equal(np.argmax(probs, 0)[decided], mask[decided])


@pytest.mark.parametrize("code", ["RAS", "PLI", "SAL"])
def test_orientation(engine, models, vol, code):
    from lungmask_b200 import orient
    _load(engine, models, 3)
    _, lps_probs = engine.apply_volume_probs(0, vol)
    native = orient.from_lps(vol, code)
    perm, flip = orient.array_transform_to_lps(code)
    mask, probs = engine.apply_volume_probs(0, native, perm, flip)
    assert probs.shape == (3,) + native.shape
    for k in range(3):
        assert np.array_equal(probs[k], orient.from_lps(lps_probs[k], code))
    assert np.array_equal(mask, engine.apply_volume_oriented(0, native, perm, flip))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_volumes(engine, models, vol, dtype):
    from lungmask_b200 import orient
    _load(engine, models, 3)
    vf = (vol.astype(np.float64) + 0.375).astype(dtype)          # fractional HU: the float path keeps them
    for pp in (True, False):
        mask, probs = engine.apply_volume_probs(0, vf, postprocess=pp)
        assert np.array_equal(mask, engine.apply_volume_float(0, vf, postprocess=pp))
        for code in ("PLI", "SAL"):
            native = orient.from_lps(vf, code)
            perm, flip = orient.array_transform_to_lps(code)
            m2, p2 = engine.apply_volume_probs(0, native, perm, flip, postprocess=pp)
            assert np.array_equal(m2, orient.from_lps(engine.apply_volume_float(0, vf, postprocess=pp), code))
            for k in range(3):
                assert np.array_equal(p2[k], orient.from_lps(probs[k], code))


def test_graphs_and_replay(engine, models, vol):
    _load(engine, models, 6)
    try:
        engine.set_option("graphs", 0)
        m0, p0 = engine.apply_volume_probs(0, vol)
        engine.set_option("graphs", 1)
        m1, p1 = engine.apply_volume_probs(0, vol)
        m2, p2 = engine.apply_volume_probs(0, vol)                # replays the captured forward
    finally:
        engine.set_option("graphs", 1)
    assert np.array_equal(m0, m1) and np.array_equal(m1, m2)
    assert np.array_equal(p0, p1) and np.array_equal(p1, p2)


def test_errors(engine, models, vol, tmp_path):
    import torch
    from lungmask_b200 import LMInferer, _native
    _load(engine, models, 3)
    with pytest.raises(_native.NativeError, match="permutation"):
        engine.apply_volume_probs(0, vol, perm=(0, 0, 1), flip=(0, 0, 0))
    with pytest.raises(TypeError):
        engine.apply_volume_probs(0, vol.astype(np.complex64))
    out = np.empty(vol.shape, np.uint8)
    probs = np.empty((3,) + vol.shape, np.float32)
    rc = _native.lib().lm_apply_volume_probs(engine._h, 0, C.c_void_p(vol.ctypes.data), 7, *vol.shape, None, None, 0,
                                             C.c_void_p(out.ctypes.data), C.c_void_p(probs.ctypes.data))
    assert rc != 0 and "dtype" in _native.lib().lm_last_error().decode()
    p6, p3 = str(tmp_path / "w6.pth"), str(tmp_path / "w3.pth")
    torch.save(models[6], p6)
    torch.save(models[3], p3)
    inf = LMInferer(modelpath=p6, fillmodel="R231", fillmodel_path=p3, batch_size=4, tqdm_disable=True)
    with pytest.raises(ValueError, match="fill model"):
        inf.apply_with_probabilities(vol)


def _nifti_header(path):
    raw = gzip.open(path, "rb").read() if path.endswith(".gz") else open(path, "rb").read()
    dim = struct.unpack_from("<8h", raw, 40)
    srow = np.asarray([struct.unpack_from("<4f", raw, 280 + 16 * r) for r in range(3)])
    return raw, dim, srow


def test_cli_probabilities(tmp_path, models, vol):
    import torch
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main

    p = str(tmp_path / "w3.pth")
    torch.save(models[3], p)
    D = np.zeros((3, 3))
    D[0, 0] = -1.0
    D[2, 1] = 1.0
    D[1, 2] = 1.0
    arr = np.ascontiguousarray(vol[:, :, ::-1].transpose(1, 0, 2))   # stored in a non-LPS orientation
    src = lio.Volume(arr, (0.75, 1.5, 0.5), (10.0, -4.0, 2.0), tuple(D.ravel()))
    in_nii = str(tmp_path / "in.nii.gz")
    lio.save_mask(in_nii, arr, src)
    image = lio.load_input_image(in_nii)
    want_mask, want_p = LMInferer(modelpath=p, batch_size=4, tqdm_disable=True).apply_with_probabilities(image)

    out_mask, out_npy, out_nii = str(tmp_path / "m.nii.gz"), str(tmp_path / "p.npy"), str(tmp_path / "p.nii.gz")
    main([in_nii, out_mask, "--modelpath", p, "--noprogress", "--batchsize", "4", "--probabilities", out_npy])
    assert np.array_equal(np.load(out_npy), want_p)
    main([in_nii, out_mask, "--modelpath", p, "--noprogress", "--batchsize", "4", "--probabilities", out_nii])
    assert np.array_equal(lio.load_input_image(out_mask).array, want_mask)
    raw, dim, srow = _nifti_header(out_nii)
    _, dim_in, srow_in = _nifti_header(in_nii)
    _, dim_m, srow_m = _nifti_header(out_mask)
    assert dim[0] == 4 and dim[4] == 3 and dim[1:4] == dim_in[1:4]
    assert np.array_equal(srow, srow_in) and np.array_equal(srow, srow_m)
    got = np.frombuffer(raw, dtype="<f4", offset=352).reshape(want_p.shape)
    assert np.array_equal(got, want_p)

    with pytest.raises(SystemExit):
        main([in_nii, out_mask, "--modelpath", p, "--probabilities", str(tmp_path / "p.mha")])
    with pytest.raises(SystemExit):
        main([in_nii, out_mask, "--modelname", "LTRCLobes_R231", "--probabilities", out_npy])
