"""GLCM and GLSZM texture features on the GPU (LMInferer.texture, lm_texture_levels_dev, lm_glcm_dev, lm_zone_sizes_dev)
against a reference written here: the level map by numpy, the 13 pair-count vectors by array slicing plus np.bincount,
the size zones by scipy.ndimage.label (26-connected) per level plus np.bincount.  Maps, counts and zones must be equal;
the features must be bit-identical to the host feature functions applied to the reference matrices."""
import json
import math

import numpy as np
import pytest
import scipy.ndimage as ndi

from lungmask_b200 import texture as tx
from oracle import synth

pytestmark = pytest.mark.gpu

FULL = np.ones((3, 3, 3), bool)


# ---- reference ---------------------------------------------------------------------------------------------------------
def ref_levels(vol, sel, bw):
    """(level map uint8, voxels, low, ng) of the ROI sel & ~isnan(vol); level map None when the ROI is empty."""
    v = np.asarray(vol)
    if v.dtype == np.float16:
        v = v.astype(np.float32)
    roi = sel & ~np.isnan(v) if v.dtype.kind == "f" else sel.copy()
    n = int(roi.sum())
    if n == 0:
        return None, 0, None, 0
    vals = v[roi]
    low, ng = tx.discretisation(float(vals.min()), float(vals.max()), bw)
    L = np.zeros(v.shape, np.uint8)
    L[roi] = tx.levels(vals, bw, low)
    return L, n, low, ng


def ref_matrices(L, ng):
    T = ng * (ng + 1) // 2
    U = np.zeros((13, T), np.int64)
    n = L.shape
    for d, off in enumerate(tx.OFFSETS):
        src = tuple(slice(max(0, -o), n[k] - max(0, o)) for k, o in enumerate(off))
        dst = tuple(slice(max(0, o), n[k] - max(0, -o)) for k, o in enumerate(off))
        a, b = L[src].astype(np.int64), L[dst].astype(np.int64)
        both = (a > 0) & (b > 0)
        i, j = np.minimum(a, b)[both], np.maximum(a, b)[both]
        U[d] = np.bincount((i - 1) * ng - (i - 1) * (i - 2) // 2 + (j - i), minlength=T)
    zones = []
    for lv in np.unique(L[L > 0]):
        lab, _ = ndi.label(L == lv, FULL)
        s, c = np.unique(np.bincount(lab.ravel())[1:], return_counts=True)
        zones += [(int(lv), int(a), int(b)) for a, b in zip(s, c)]
    return U, np.array(zones, np.int64).reshape(-1, 3)


def reference(vol, mask, bw):
    """{row: (level map, voxels, low, ng, U, zones)} for every label value in the mask and "lung"."""
    out = {}
    for row in [int(x) for x in np.unique(mask) if x] + ["lung"]:
        sel = (mask > 0) if row == "lung" else (mask == row)
        L, n, low, ng = ref_levels(vol, sel, bw)
        U, zones = ref_matrices(L, ng) if n else (None, None)
        out[row] = (L, n, low, ng, U, zones)
    return out


def _features_json(row):
    return json.dumps({"glcm": row.glcm, "glszm": row.glszm})   # NaN-safe, bit-exact through repr


def check(res, want, bw):
    for row, (L, n, low, ng, U, zones) in want.items():
        r = res[row]
        assert (r.voxels, r.low, r.n_levels, r.bin_width) == (n, low, ng, bw), (row, r.voxels, r.low, r.n_levels)
        if n == 0:
            continue
        np.testing.assert_array_equal(r.glcm_counts, U, err_msg=str(row))
        np.testing.assert_array_equal(r.zones, zones, err_msg=str(row))
        expect = tx.build_row(256 if row == "lung" else row, r.name, n, bw, low, ng, U, zones)
        assert _features_json(r) == _features_json(expect), row
    for r in res.rows:
        if r.label not in want or want[r.label][1] == 0:
            assert r.voxels == 0 and r.n_levels == 0 and all(math.isnan(v) for v in r.glcm.values())


def check_level_maps(eng, vol, mask, want, bw, dtype_code):
    """lm_texture_levels_dev of every row equals the numpy level map exactly."""
    import torch
    tv, tm = _cuda(vol), _cuda(mask)
    lev = torch.full(mask.shape, 77, dtype=torch.uint8, device="cuda:0")
    for row, (L, n, low, ng, _, _) in want.items():
        if n == 0:
            continue
        eng.texture_levels_dev(tv.data_ptr(), dtype_code, tm.data_ptr(), mask.shape, 256 if row == "lung" else row, low, bw, ng,
                               lev.data_ptr())
        np.testing.assert_array_equal(lev.cpu().numpy(), L, err_msg=str(row))


@pytest.fixture(scope="module")
def inf():
    import os
    import tempfile
    import torch
    from lungmask_b200 import LMInferer
    fd, path = tempfile.mkstemp(suffix=".pth")
    os.close(fd)
    try:
        torch.save(synth.random_state_dict(3, seed=47, head_gain=0.3), path)
        return LMInferer(modelpath=path, batch_size=4, tqdm_disable=True)
    finally:
        os.remove(path)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _bytes(t):
    return t.cpu().numpy().tobytes()


def both_paths(inf, vol, mask, **kw):
    """texture() on numpy arrays and on CUDA tensors: identical to_dict(), inputs unmodified; returns the numpy one."""
    a = inf.texture(vol, mask, **kw)
    tv, tm = _cuda(vol), _cuda(mask)
    bv, bm = tv.clone(), tm.clone()
    b = inf.texture(tv, tm, **kw)
    assert _bytes(tv) == _bytes(bv) and _bytes(tm) == _bytes(bm), "an input tensor was modified"
    assert json.dumps(a.to_dict()) == json.dumps(b.to_dict())
    return a


@pytest.fixture(scope="module")
def lungs():
    """30x96x112 int16 phantom with a two-lung ellipsoid mask; and the same lungs split into five lobes."""
    S, H, W = 30, 96, 112
    vol = synth.phantom(S, H, W, seed=31)
    z, y, x = np.ogrid[:S, :H, :W]
    mask = np.zeros((S, H, W), np.uint8)
    for label, cx in ((1, 0.32), (2, 0.68)):
        mask[((z - S / 2) / (0.45 * S)) ** 2 + ((y - 0.5 * H) / (0.3 * H)) ** 2 + ((x - cx * W) / (0.15 * W)) ** 2 <= 1.0] = label
    lobes = mask.copy()
    lobes[(mask == 1) & (z < S // 2)] = 3
    lobes[(mask == 1) & (z >= S // 2) & (y < H // 2)] = 4
    lobes[(mask == 1) & (z >= S // 2) & (y >= H // 2)] = 5
    return vol, mask, lobes


DTYPE_CODES = {np.dtype(np.int16): 0, np.dtype(np.float32): 1, np.dtype(np.float64): 2}


@pytest.mark.parametrize("dtype", [np.int16, np.float32, np.float64])
@pytest.mark.parametrize("which", ["lungs", "lobes"])
def test_phantom(inf, lungs, dtype, which):
    vol, mask, lobes = lungs
    m = mask if which == "lungs" else lobes
    rng = np.random.default_rng(71)
    v = vol if dtype == np.int16 else (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(dtype)
    if dtype != np.int16:
        v[rng.random(v.shape) < 0.03] = np.nan
        edge = np.flatnonzero(m == 2)[:2]   # a bin edge and one ulp below it
        v.flat[edge] = (-850.0, np.nextafter(dtype(-850.0), dtype(-2000.0)))
    want = reference(v, m, 25)
    res = both_paths(inf, v, m)
    check(res, want, 25)
    # the labels in the mask and the model's labels 1..2 (label 1 is absent from the lobe mask: 0 voxels)
    assert [r.label for r in res.rows] == sorted({int(x) for x in np.unique(m) if x} | {1, 2}) + ["lung"]
    assert 20 < res["lung"].n_levels <= 90   # the shared-memory GLCM path
    check_level_maps(inf.engine, v, m, want, 25, DTYPE_CODES[np.dtype(dtype)])


def test_float16_tensor(inf, lungs):
    import torch
    vol, mask, _ = lungs
    rng = np.random.default_rng(72)
    v = (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(np.float32)
    v[rng.random(v.shape) < 0.02] = np.nan
    for dt in (torch.float16, torch.bfloat16):
        h = torch.from_numpy(v).to(dt)
        got = inf.texture(h.to("cuda:0"), _cuda(mask))
        check(got, reference(h.float().numpy(), mask, 25), 25)
        assert json.dumps(inf.texture(h, mask).to_dict()) == json.dumps(got.to_dict())   # CPU tensor: numpy path


def test_random_labels_touch_every_face_band_path(inf):
    """Random labels over the whole array (every ROI touches all six faces) and values spanning ~150 levels at bw 4:
    the GLCM's band + global-atomic path."""
    rng = np.random.default_rng(73)
    shape = (17, 45, 70)
    mask = rng.integers(0, 4, shape).astype(np.uint8)
    mask[rng.random(shape) < 0.5] = 1
    vol = np.round(rng.normal(-300, 120, shape)).clip(-600, -1).astype(np.int16)
    want = reference(vol, mask, 4)
    assert all(91 <= want[r][3] <= 255 for r in want)
    res = both_paths(inf, vol, mask, bin_width=4)
    check(res, want, 4)
    f = vol.astype(np.float32) + rng.uniform(0, 1, shape).astype(np.float32)
    f[rng.random(shape) < 0.05] = np.nan
    check(both_paths(inf, f, mask, bin_width=4), reference(f, mask, 4), 4)
    check_level_maps(inf.engine, vol, mask, want, 4, 0)


def test_exactly_255_levels_and_single_voxel(inf):
    rng = np.random.default_rng(74)
    shape = (9, 33, 41)
    vol = rng.integers(-100, 155, shape).astype(np.int16)
    vol[0, 0, 0], vol[-1, -1, -1] = -100, 154
    mask = np.ones(shape, np.uint8)
    mask[4, 16, 20] = 2                                   # a single-voxel ROI
    want = reference(vol, mask, 1)
    assert want["lung"][3] == 255 and want[2][1] == 1
    res = both_paths(inf, vol, mask, bin_width=1)
    check(res, want, 1)
    assert all(math.isnan(v) for v in res[2].glcm.values()) and res[2].glszm["ZonePercentage"] == 1.0
    with pytest.raises(ValueError, match="row lung .*more than 255"):
        inf.texture(np.where(mask == 1, vol, 155).astype(np.int16), mask, bin_width=1)


def test_flip_and_transpose_within_1e12(inf, lungs):
    vol, _, lobes = lungs
    a = inf.texture(vol, lobes)
    for f in (lambda x: x[::-1], lambda x: x[:, :, ::-1], lambda x: x.transpose(0, 2, 1)):
        b = inf.texture(np.ascontiguousarray(f(vol)), np.ascontiguousarray(f(lobes)))
        for ra, rb in zip(a.rows, b.rows):
            assert ra.label == rb.label and ra.voxels == rb.voxels
            for fa, fb in ((ra.glcm, rb.glcm), (ra.glszm, rb.glszm)):
                for k, va in fa.items():
                    vb = fb[k]
                    same = (math.isnan(va) and math.isnan(vb)) or abs(va - vb) <= 1e-12 * max(1.0, abs(va))
                    assert same, (ra.label, k, va, vb)


def test_errors(inf, lungs):
    from lungmask_b200 import _native
    vol, mask, _ = lungs
    eng = inf.engine
    f = vol.astype(np.float32)
    f.flat[np.flatnonzero(mask == 2)[5]] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        inf.texture(f, mask)
    with pytest.raises(ValueError):
        inf.texture(vol, mask, bin_width=0)
    with pytest.raises(TypeError):
        inf.texture(vol, mask, bin_width=2.5)
    tv, tm = _cuda(vol), _cuda(mask)
    want = reference(vol, mask, 25)
    L, n, low, ng, U, _ = want["lung"]
    import torch
    lev = torch.empty(mask.shape, dtype=torch.uint8, device="cuda:0")
    # n_levels below the largest level: an error, never a wrong map or wrong counts
    with pytest.raises(_native.NativeError, match="level outside"):
        eng.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), mask.shape, 256, low, 25, ng - 1, lev.data_ptr())
    with pytest.raises(_native.NativeError, match="level outside"):
        eng.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), mask.shape, 256, low + 25, 25, ng, lev.data_ptr())
    tL = _cuda(L)
    with pytest.raises(_native.NativeError, match="level outside"):
        eng.glcm_dev(tL.data_ptr(), mask.shape, ng - 1)
    np.testing.assert_array_equal(eng.glcm_dev(tL.data_ptr(), mask.shape, ng), U)
    tf = _cuda(f)
    with pytest.raises(_native.NativeError, match="non-finite"):
        eng.texture_levels_dev(tf.data_ptr(), 1, tm.data_ptr(), mask.shape, 2, -2000, 25, 255, lev.data_ptr())
    with pytest.raises(_native.NativeError, match="aligned"):
        eng.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), (1, 1, 8), 256, low, 25, ng, lev.data_ptr() + 1)
    with pytest.raises(_native.NativeError, match="row"):
        eng.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), mask.shape, 0, low, 25, ng, lev.data_ptr())
    with pytest.raises(_native.NativeError, match="bin_width"):
        eng.texture_levels_dev(tv.data_ptr(), 0, tm.data_ptr(), mask.shape, 1, low, 0, ng, lev.data_ptr())
    with pytest.raises(_native.NativeError, match="n_levels"):
        eng.glcm_dev(tL.data_ptr(), mask.shape, 256)
    with pytest.raises(_native.NativeError, match="2\\^32"):
        eng.zone_sizes_dev(tL.data_ptr(), (65536, 65536, 1))
    # the engine still works after the refusals
    check(inf.texture(tv, tm), want, 25)


def test_zone_sizes_dev_rows(inf, lungs):
    vol, mask, lobes = lungs
    L, n, low, ng, _, zones = reference(vol, lobes, 25)["lung"]
    res = inf.engine.zone_sizes_dev(_cuda(L).data_ptr(), L.shape)
    assert res["n_pairs"][0] == 0 and int(res["n_pairs"].sum()) == zones.shape[0]
    np.testing.assert_array_equal(tx.zones_from_native(res), zones)
    assert int((res["sizes"] * res["counts"]).sum()) == n


@pytest.mark.parametrize("ext", ["json", "csv"])
def test_cli(tmp_path, ext):
    import csv
    import torch
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    wpath = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=48, head_gain=0.3), wpath)
    vol = synth.phantom(6, 160, 176, seed=24)
    src = lio.Volume(vol, (0.75, 0.5, 1.5))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = str(tmp_path / ("texture." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", wpath, "--noprogress", "--batchsize", "4", "--texture", out,
          "--texture-bin-width", "20"])
    inf = LMInferer(modelpath=wpath, tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.texture(v, inf.apply(v), bin_width=20)
    if ext == "json":
        got = json.load(open(out))
        assert got == json.loads(json.dumps(want.to_dict()))
        assert got["bin_width"] == 20
    else:
        rows = list(csv.DictReader(open(out)))
        assert [r["label"] for r in rows] == [str(r.label) for r in want.rows]
        for r, w in zip(rows, want.rows):
            assert int(r["voxels"]) == w.voxels and int(r["n_levels"]) == w.n_levels
            for k in tx.GLCM_FEATURES:
                assert float(r["glcm_" + k]) == w.glcm[k] or math.isnan(w.glcm[k])
