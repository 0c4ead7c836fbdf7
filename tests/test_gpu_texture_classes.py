"""GLRLM, GLDM and NGTDM on the GPU (LMInferer.texture(classes=...), lm_glrlm_dev, lm_neighbour_counts_dev) against the
numpy references of _texture_ref (run positions along each direction; 26 shifted slices of the padded map) on the level
maps of test_gpu_texture's reference.  Every matrix must be equal, every feature bit-identical to the host functions
applied to the reference matrices, and the GLCM / GLSZM part identical to texture() with the default classes."""
import json
import math

import numpy as np
import pytest

import test_gpu_texture as base
from _texture_ref import glrlm_ref, neighbour_ref
from lungmask_b200 import texture as tx
from oracle import synth

pytestmark = pytest.mark.gpu

ALL = tx.CLASSES
SHORT_RUN_WORDS = 53235   # the shared run counters of lm_glrlm_dev: lengths <= 53235 // (13 Ng) are privatised


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


def _json(row):
    return json.dumps({c: getattr(row, c) for c in ALL})   # NaN-safe, bit-exact through repr


def check(res, vol, mask, bw, alpha=0):
    """res (texture(classes=ALL)) against the reference of every row; returns the reference."""
    want = base.reference(vol, mask, bw)
    base.check(res, want, bw)
    assert res.classes == ALL and res.gldm_alpha == alpha
    for row, (L, n, low, ng, U, zones) in want.items():
        r = res[row]
        if n == 0:
            continue
        P = glrlm_ref(L, ng)
        G, N, A = neighbour_ref(L, ng, alpha)
        np.testing.assert_array_equal(r.glrlm_runs, tx.runs_from_counts(P), err_msg=str(row))
        for got, ref in ((r.gldm_counts, G), (r.ngtdm_counts, N), (r.ngtdm_sums, A)):
            np.testing.assert_array_equal(got, ref, err_msg=str(row))
        expect = tx.build_row(256 if row == "lung" else row, r.name, n, bw, low, ng, U, zones, ALL, P, (G, N, A))
        assert _json(r) == _json(expect), row
    for r in res.rows:
        if r.label not in want or want[r.label][1] == 0:
            assert r.voxels == 0 and all(math.isnan(v) for c in ALL for v in getattr(r, c).values())
    return want


def check_dev(eng, want, alpha=0):
    """lm_glrlm_dev / lm_neighbour_counts_dev on every reference level map: the dense matrices."""
    for row, (L, n, low, ng, U, zones) in want.items():
        if n == 0:
            continue
        tL = base._cuda(L)
        np.testing.assert_array_equal(eng.glrlm_dev(tL.data_ptr(), L.shape, ng), glrlm_ref(L, ng), err_msg=str(row))
        for got, ref in zip(eng.neighbour_counts_dev(tL.data_ptr(), L.shape, ng, alpha), neighbour_ref(L, ng, alpha)):
            np.testing.assert_array_equal(got, ref, err_msg=str(row))


def same_default_part(a, b):
    """The GLCM / GLSZM part of texture(classes=ALL) `a` is that of texture() `b`."""
    for ra, rb in zip(a.rows, b.rows):
        assert json.dumps({k: ra.to_dict()[k] for k in rb.to_dict()}) == json.dumps(rb.to_dict())
        np.testing.assert_array_equal(ra.glcm_counts, rb.glcm_counts)


@pytest.mark.parametrize("alpha", [0, 2])
@pytest.mark.parametrize("dtype", [np.int16, np.float32, np.float64])
@pytest.mark.parametrize("which", ["lungs", "lobes"])
def test_phantom(inf, lungs, dtype, which, alpha):
    vol, mask, lobes = lungs
    m = mask if which == "lungs" else lobes
    rng = np.random.default_rng(81)
    v = vol if dtype == np.int16 else (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(dtype)
    if dtype != np.int16:
        v[rng.random(v.shape) < 0.03] = np.nan
    res = base.both_paths(inf, v, m, classes=ALL, gldm_alpha=alpha)
    want = check(res, v, m, 25, alpha)
    same_default_part(res, inf.texture(v, m))
    assert 20 < res["lung"].n_levels <= 90
    if dtype == np.int16:
        check_dev(inf.engine, want, alpha)


def test_float16_tensor(inf, lungs):
    import torch
    vol, mask, _ = lungs
    rng = np.random.default_rng(82)
    v = (vol + rng.uniform(-0.5, 0.5, vol.shape)).astype(np.float32)
    v[rng.random(v.shape) < 0.02] = np.nan
    for dt in (torch.float16, torch.bfloat16):
        h = torch.from_numpy(v).to(dt)
        got = inf.texture(h.to("cuda:0"), base._cuda(mask), classes=ALL)
        check(got, h.float().numpy(), mask, 25)
        assert json.dumps(inf.texture(h, mask, classes=ALL).to_dict()) == json.dumps(got.to_dict())


def test_random_labels_touch_every_face_global_runs(inf):
    """Random labels over the whole array, ~150 levels at bw 4, and three constant rows of full-length x-runs: runs
    longer than the shared range go to global atomics."""
    rng = np.random.default_rng(83)
    shape = (17, 45, 70)
    mask = rng.integers(0, 4, shape).astype(np.uint8)
    mask[rng.random(shape) < 0.5] = 1
    vol = np.round(rng.normal(-300, 120, shape)).clip(-600, -1).astype(np.int16)
    mask[:, :3, :] = 1
    vol[:, :3, :] = -300
    res = base.both_paths(inf, vol, mask, bin_width=4, classes=ALL, gldm_alpha=2)
    want = check(res, vol, mask, 4, alpha=2)
    for row in (1, "lung"):
        ng = want[row][3]
        assert 91 <= ng <= 255
        assert res[row].glrlm_runs[:, 2].max() > SHORT_RUN_WORDS // (13 * ng), row
    check_dev(inf.engine, want, alpha=2)


def test_exactly_255_levels_and_single_voxel(inf):
    rng = np.random.default_rng(84)
    shape = (9, 33, 41)
    vol = rng.integers(-100, 155, shape).astype(np.int16)
    vol[0, 0, 0], vol[-1, -1, -1] = -100, 154
    mask = np.ones(shape, np.uint8)
    mask[4, 16, 20] = 2                                   # a single-voxel ROI
    res = base.both_paths(inf, vol, mask, bin_width=1, classes=ALL)
    want = check(res, vol, mask, 1)
    assert want["lung"][3] == 255 and want[2][1] == 1
    one = res[2]
    assert all(math.isnan(v) for v in one.ngtdm.values())
    assert one.glrlm["RunPercentage"] == 1.0 and one.gldm["SmallDependenceEmphasis"] == 1.0
    assert one.glrlm_runs.tolist() == [[d, 1, 1, 1] for d in range(13)]
    check_dev(inf.engine, want)


@pytest.mark.parametrize("shape", [(37, 45, 600), (300, 3, 2)])
def test_uniform_roi_fills_the_array(inf, shape):
    """One level everywhere: every run spans the array, the longest walks."""
    vol = np.full(shape, -800, np.int16)
    mask = np.ones(shape, np.uint8)
    res = base.both_paths(inf, vol, mask, classes=ALL)
    want = check(res, vol, mask, 25)
    r = res["lung"]
    assert r.n_levels == 1 and r.glrlm_runs[0].tolist() == [0, 1, shape[2], shape[0] * shape[1]]
    assert r.ngtdm["Coarseness"] == 1e6 and r.gldm_counts[0, 26] == (shape[0] - 2) * (shape[1] - 2) * (shape[2] - 2)
    check_dev(inf.engine, want)


def test_flip_and_transpose(inf, lungs):
    """GLDM / NGTDM matrices are identical under flips and transposes; GLRLM features agree to 1e-12 (the directions are
    permuted)."""
    vol, _, lobes = lungs
    a = inf.texture(vol, lobes, classes=ALL, gldm_alpha=2)
    for f in (lambda x: x[::-1], lambda x: x[:, :, ::-1], lambda x: x.transpose(0, 2, 1), lambda x: x.transpose(2, 1, 0)):
        b = inf.texture(np.ascontiguousarray(f(vol)), np.ascontiguousarray(f(lobes)), classes=ALL, gldm_alpha=2)
        for ra, rb in zip(a.rows, b.rows):
            assert ra.label == rb.label and ra.voxels == rb.voxels
            if not ra.voxels:
                continue
            for k in ("gldm_counts", "ngtdm_counts", "ngtdm_sums"):
                np.testing.assert_array_equal(getattr(ra, k), getattr(rb, k))
            assert json.dumps([ra.gldm, ra.ngtdm]) == json.dumps([rb.gldm, rb.ngtdm])
            assert int(ra.glrlm_runs[:, 3].sum()) == int(rb.glrlm_runs[:, 3].sum())
            for k, va in ra.glrlm.items():
                vb = rb.glrlm[k]
                assert abs(va - vb) <= 1e-12 * max(1.0, abs(va)), (ra.label, k, va, vb)


def test_errors(inf, lungs):
    from lungmask_b200 import _native
    vol, mask, _ = lungs
    eng = inf.engine
    for bad, err in (({"classes": ("glcm", "glrlmx")}, ValueError), ({"classes": ()}, ValueError),
                     ({"classes": "glrlm"}, TypeError), ({"gldm_alpha": -1}, ValueError), ({"gldm_alpha": 0.5}, TypeError)):
        with pytest.raises(err):
            inf.texture(vol, mask, **bad)
    want = base.reference(vol, mask, 25)
    L, n, low, ng, U, _ = want["lung"]
    tL = base._cuda(L)
    # n_levels below the largest level: an error, never wrong counts
    with pytest.raises(_native.NativeError, match="level outside"):
        eng.glrlm_dev(tL.data_ptr(), L.shape, ng - 1)
    with pytest.raises(_native.NativeError, match="level outside"):
        eng.neighbour_counts_dev(tL.data_ptr(), L.shape, ng - 1, 0)
    for call in (lambda: eng.glrlm_dev(tL.data_ptr(), L.shape, 256),
                 lambda: eng.neighbour_counts_dev(tL.data_ptr(), L.shape, 256, 0),
                 lambda: eng.glrlm_dev(tL.data_ptr(), L.shape, 0)):
        with pytest.raises(_native.NativeError, match="n_levels"):
            call()
    with pytest.raises(_native.NativeError, match="alpha"):
        eng.neighbour_counts_dev(tL.data_ptr(), L.shape, ng, -1)
    with pytest.raises(_native.NativeError, match="2\\^32"):
        eng.glrlm_dev(tL.data_ptr(), (4096, 1024, 1024), ng)
    with pytest.raises(_native.NativeError, match="2\\^32"):
        eng.neighbour_counts_dev(tL.data_ptr(), (4096, 1024, 1024), ng, 0)
    with pytest.raises(_native.NativeError, match="NULL"):
        eng.glrlm_dev(0, L.shape, ng)
    # the engine still works after the refusals
    check(inf.texture(base._cuda(vol), base._cuda(mask), classes=ALL), vol, mask, 25)
    np.testing.assert_array_equal(eng.glrlm_dev(tL.data_ptr(), L.shape, ng), glrlm_ref(L, ng))


@pytest.mark.parametrize("ext", ["json", "csv"])
def test_cli(tmp_path, ext):
    import csv
    import torch
    from lungmask_b200 import LMInferer, io as lio
    from lungmask_b200.__main__ import main
    wpath = str(tmp_path / "w3.pth")
    torch.save(synth.random_state_dict(3, seed=49, head_gain=0.3), wpath)
    vol = synth.phantom(6, 160, 176, seed=25)
    src = lio.Volume(vol, (0.75, 0.5, 1.5))
    inp = str(tmp_path / "in.mha")
    lio.save_mask(inp, vol, src)
    out = str(tmp_path / ("texture." + ext))
    main([inp, str(tmp_path / "mask.nii.gz"), "--modelpath", wpath, "--noprogress", "--batchsize", "4", "--texture", out,
          "--texture-bin-width", "20", "--texture-classes", "ngtdm,glrlm,gldm"])
    inf = LMInferer(modelpath=wpath, tqdm_disable=True, batch_size=4)
    v = lio.load_input_image(inp)
    want = inf.texture(v, inf.apply(v), bin_width=20, classes=("glrlm", "gldm", "ngtdm"))
    if ext == "json":
        got = json.load(open(out))
        assert got == json.loads(json.dumps(want.to_dict()))
        assert got["classes"] == ["glrlm", "gldm", "ngtdm"] and got["gldm_alpha"] == 0
        assert all("glcm" not in r and "glrlm" in r for r in got["rows"])
    else:
        rows = list(csv.DictReader(open(out)))
        assert [r["label"] for r in rows] == [str(r.label) for r in want.rows]
        assert not any(k.startswith(("glcm_", "glszm_")) for k in rows[0])
        for r, w in zip(rows, want.rows):
            for c, names in (("glrlm", tx.GLRLM_FEATURES), ("gldm", tx.GLDM_FEATURES), ("ngtdm", tx.NGTDM_FEATURES)):
                for k in names:
                    assert float(r[c + "_" + k]) == getattr(w, c)[k] or math.isnan(getattr(w, c)[k])
